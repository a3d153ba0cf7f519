"""A ROS1 bag (format 2.0) reader: the messages of chosen topics in record-time order, with the standard library and numpy only.

The format: the file starts with "#ROSBAG V2.0\\n"; then records of {u32 header_len, header, u32 data_len, data}. A header is a list of
{u32 len, "name=value"} fields with little-endian binary values; its "op" field is the record type (OP_* below). Messages sit in chunk
records (compression none / bz2 / lz4); every chunk is followed by one index-data record per connection it holds, listing each message's
record time and offset inside the uncompressed chunk. Connections and chunk infos follow the last chunk, at the bag header's index_pos.

Delivery is that of `rosbag play`: by record time across all chosen connections, ties broken by file position. The file is memory-mapped;
a chunk is decompressed when its first message is delivered and released after its last one. A bag whose recording was cut off (no
index, or a last chunk that ends early) is read chunk by chunk up to its last complete message record, with a warning.
"""
from __future__ import annotations

import bz2
import mmap
import os
import struct
import warnings

import numpy as np

from . import rosmsg

MAGIC = b"#ROSBAG V2.0\n"
OP_MSG_DATA, OP_BAG_HEADER, OP_INDEX_DATA, OP_CHUNK, OP_CHUNK_INFO, OP_CONNECTION = 0x02, 0x03, 0x04, 0x05, 0x06, 0x07


class BagError(RuntimeError):
    pass


class BagWarning(UserWarning):
    pass


def parse_header(buf, pos: int, end: int) -> dict:
    """The fields of a record header buf[pos:end] as {name: bytes value}."""
    out = {}
    while pos < end:
        if pos + 4 > end:
            raise BagError(f"header field at byte {pos} overruns its header")
        (n,) = struct.unpack_from("<I", buf, pos)
        pos += 4
        if pos + n > end:
            raise BagError(f"header field at byte {pos - 4} overruns its header")
        field = bytes(buf[pos:pos + n])
        eq = field.find(b"=")
        if eq < 0:
            raise BagError(f"header field at byte {pos - 4} has no '='")
        out[field[:eq].decode("latin-1")] = field[eq + 1:]
        pos += n
    return out


def _u32(v: bytes) -> int:
    return struct.unpack("<I", v)[0]


def _u64(v: bytes) -> int:
    return struct.unpack("<Q", v)[0]


def _time_ns(v: bytes) -> int:
    sec, nsec = struct.unpack("<II", v)
    return sec * 1_000_000_000 + nsec


def read_record(buf, pos: int, size: int):
    """The record at pos: (header dict, data_start, data_len, next_pos), or None when it does not fit in the first `size` bytes."""
    if pos + 4 > size:
        return None
    (hl,) = struct.unpack_from("<I", buf, pos)
    if pos + 4 + hl + 4 > size:
        return None
    hdr = parse_header(buf, pos + 4, pos + 4 + hl)
    (dl,) = struct.unpack_from("<I", buf, pos + 4 + hl)
    start = pos + 8 + hl
    if start + dl > size:
        return None
    return hdr, start, dl, start + dl


class Message:
    """One delivered message: topic, msg type, record time (sec, nsec) and its serialized data (a zero-copy view where possible)."""
    __slots__ = ("topic", "type", "sec", "nsec", "data")

    def __init__(self, topic, type_, sec, nsec, data):
        self.topic, self.type, self.sec, self.nsec, self.data = topic, type_, sec, nsec, data

    @property
    def time(self) -> float:
        return self.sec + 1e-9 * self.nsec


class _Chunk:
    __slots__ = ("pos", "compression", "size", "start", "length", "complete", "entries")

    def __init__(self, pos, compression, size, start, length, complete):
        self.pos, self.compression, self.size, self.start, self.length, self.complete = pos, compression, size, start, length, complete
        self.entries = None   # [(conn, time_ns, offset)] from the chunk's index-data records; None -> not indexed


class Bag:
    """bag = Bag(path); bag.topics() -> {topic: type}; for m in bag.messages({topic: (type, ...)}): ..."""
    format = "ros1"     # the serialization of its messages (rosmsg.decoders)

    def __init__(self, path: str):
        self.path = path
        self._f = open(path, "rb")
        size = os.fstat(self._f.fileno()).st_size
        if size < len(MAGIC):
            self._f.close()
            raise BagError(f"{path}: not a ROS1 bag (file of {size} bytes)")
        self._mm = mmap.mmap(self._f.fileno(), 0, access=mmap.ACCESS_READ)
        head = bytes(self._mm[:len(MAGIC)])
        if head != MAGIC:
            self.close()
            raise BagError(f"{path}: not a ROS1 bag v2.0 (it starts with {head!r})")
        self.size = size
        self.connections = {}    # conn id -> dict(topic, type, md5sum, message_definition)
        self.chunks = []
        self.truncated = False
        self._scan()

    def close(self):
        if getattr(self, "_mm", None) is not None:
            try:
                self._mm.close()
            except BufferError:   # a delivered message still views the map; it is unmapped when the last view goes
                pass
            self._mm = None
        if getattr(self, "_f", None) is not None:
            self._f.close()
            self._f = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- the top-level pass: chunk positions, index data, connections ----
    def _scan(self):
        mm, pos, index_pos, chunk = self._mm, len(MAGIC), 0, None
        while pos < self.size:
            rec = read_record(mm, pos, self.size)
            if rec is None:
                self.truncated = True
                break
            hdr, start, dl, nxt = rec
            if "op" not in hdr:
                raise BagError(f"{self.path}: record at byte {pos} has no op field")
            op = hdr["op"][0]
            if op == OP_BAG_HEADER:
                index_pos = _u64(hdr["index_pos"])
            elif op == OP_CHUNK:
                comp = hdr["compression"].decode()
                chunk = _Chunk(pos, comp, _u32(hdr["size"]), start, dl, True)
                self.chunks.append(chunk)
            elif op == OP_INDEX_DATA:
                if chunk is None:
                    raise BagError(f"{self.path}: index data at byte {pos} precedes every chunk")
                if _u32(hdr["ver"]) != 1:
                    raise BagError(f"{self.path}: index data at byte {pos} has version {_u32(hdr['ver'])}, not 1")
                conn, count = _u32(hdr["conn"]), _u32(hdr["count"])
                if dl != 12 * count:
                    raise BagError(f"{self.path}: index data at byte {pos} holds {dl} bytes for {count} entries")
                a = np.frombuffer(mm, np.uint32, 3 * count, start).reshape(count, 3).astype(np.int64)
                if chunk.entries is None:
                    chunk.entries = []
                chunk.entries.extend(zip([conn] * count, (a[:, 0] * 1_000_000_000 + a[:, 1]).tolist(), a[:, 2].tolist()))
            elif op == OP_CONNECTION:
                self._add_connection(hdr, mm, start, dl, pos)
            pos = nxt
        if self.truncated:
            # a chunk cut off in its data: keep it, read up to its last complete message record
            rec = self._partial_chunk(pos)
            if rec is not None:
                self.chunks.append(rec)
        if self.truncated or index_pos == 0 or index_pos >= self.size or any(c.entries is None for c in self.chunks):
            # no complete index (the connection records sit after the last chunk): every chunk is read itself, in file order
            for c in self.chunks:
                c.entries = self._chunk_entries(c)
            what = "ends inside a record" if self.truncated else "has no index"
            warnings.warn(f"{self.path}: the bag {what} (a recording that was cut off?); read sequentially up to its last complete "
                          f"message record ({len(self.chunks)} chunks)", BagWarning, stacklevel=3)
        unknown = {e[0] for c in self.chunks for e in c.entries} - set(self.connections)
        if unknown:
            raise BagError(f"{self.path}: messages of connections {sorted(unknown)} that no connection record describes")

    def _partial_chunk(self, pos):
        mm = self._mm
        if pos + 4 > self.size:
            return None
        (hl,) = struct.unpack_from("<I", mm, pos)
        if pos + 8 + hl > self.size:
            return None
        hdr = parse_header(mm, pos + 4, pos + 4 + hl)
        if hdr.get("op", b"\0")[0] != OP_CHUNK:
            return None
        start = pos + 8 + hl
        return _Chunk(pos, hdr["compression"].decode(), _u32(hdr["size"]), start, self.size - start, False)

    def _add_connection(self, hdr, buf, start, dl, pos):
        conn = _u32(hdr["conn"])
        fields = parse_header(buf, start, start + dl)
        if "type" not in fields:
            raise BagError(f"{self.path}: connection record at byte {pos} has no type")
        self.connections[conn] = dict(topic=hdr["topic"].decode(), type=fields["type"].decode(),
                                      md5sum=fields.get("md5sum", b"").decode(), message_definition=fields.get("message_definition", b"").decode())

    def _chunk_data(self, c: _Chunk):
        """The uncompressed data of a chunk (a view into the map for uncompressed chunks)."""
        raw = memoryview(self._mm)[c.start:c.start + c.length]
        if c.compression == "none":
            return raw
        if c.compression == "bz2":
            d = bz2.BZ2Decompressor()
            try:
                return memoryview(d.decompress(raw))
            except (OSError, EOFError, ValueError) as e:
                if c.complete:
                    raise BagError(f"{self.path}: chunk at byte {c.pos}: bz2 data is corrupt ({e})") from None
                return memoryview(b"")
        if c.compression == "lz4":
            raise BagError(f"{self.path}: chunk at byte {c.pos} is lz4-compressed, which this reader does not support; "
                           f"run `rosbag decompress {os.path.basename(self.path)}` (or `rosbag compress --bz2`) first")
        raise BagError(f"{self.path}: chunk at byte {c.pos} has unknown compression {c.compression!r}")

    def _chunk_entries(self, c: _Chunk):
        """The message records of a chunk without an index, read in order up to the last complete one; connection records inside
        the chunk are taken in."""
        data = self._chunk_data(c)
        n = len(data) if c.complete else min(len(data), c.size)
        out, pos = [], 0
        while pos < n:
            rec = read_record(data, pos, n)
            if rec is None:
                if c.complete:
                    raise BagError(f"{self.path}: chunk at byte {c.pos}: record at offset {pos} overruns the chunk")
                break
            hdr, start, dl, nxt = rec
            op = hdr["op"][0]
            if op == OP_MSG_DATA:
                out.append((_u32(hdr["conn"]), _time_ns(hdr["time"]), pos))
            elif op == OP_CONNECTION:
                self._add_connection(hdr, data, start, dl, c.pos)
            pos = nxt
        return out

    # ---- the public side ----
    def topics(self) -> dict:
        """{topic: message type} of every connection."""
        return {c["topic"]: c["type"] for c in self.connections.values()}

    def _describe(self) -> str:
        t = self.topics()
        return "; ".join(f"{k} [{v}]" for k, v in sorted(t.items())) or "(none)"

    def check_topics(self, wanted: dict) -> dict:
        """wanted {topic: accepted type or tuple of types}. Raises BagError naming the bag's topics for a missing topic or a topic of
        another type, and a livox_ros_driver2/CustomMsg connection whose definition differs from livox_ros_driver/CustomMsg (naming the
        first field that differs). Returns {conn id: topic} of the chosen connections."""
        out = {}
        for topic, types in wanted.items():
            types = (types,) if isinstance(types, str) else tuple(types)
            conns = {k: c for k, c in self.connections.items() if c["topic"] == topic}
            if not conns:
                raise BagError(f"{self.path}: no topic {topic!r} in the bag; it has: {self._describe()}")
            for k, c in conns.items():
                if c["type"] not in types:
                    raise BagError(f"{self.path}: topic {topic!r} carries {c['type']}, expected {' or '.join(types)}; the bag has: "
                                   f"{self._describe()}")
                why = rosmsg.definition_mismatch(c["type"], c["message_definition"])
                if why is not None:
                    raise BagError(f"{self.path}: topic {topic!r} carries {c['type']}, whose message_definition differs from "
                                   f"{rosmsg.LIVOX_TYPE}: {why}")
                out[k] = topic
        return out

    def count(self, wanted: dict) -> int:
        conns = self.check_topics(wanted)
        return sum(1 for c in self.chunks for e in c.entries if e[0] in conns)

    def messages(self, wanted: dict):
        """Yield the Message of every record of the chosen topics in (record time, file position) order."""
        conns = self.check_topics(wanted)
        order = []
        for ci, c in enumerate(self.chunks):
            order.extend((t, ci, off, conn) for conn, t, off in c.entries if conn in conns)
        order.sort()
        last_use = {}
        for i, (_, ci, _, _) in enumerate(order):
            last_use[ci] = i
        live = {}
        for i, (t, ci, off, conn) in enumerate(order):
            data = live.get(ci)
            if data is None:
                data = live[ci] = self._chunk_data(self.chunks[ci])
            rec = read_record(data, off, len(data))
            if rec is None:
                raise BagError(f"{self.path}: chunk at byte {self.chunks[ci].pos}: message record at offset {off} overruns the chunk")
            hdr, start, dl, _ = rec
            if hdr["op"][0] != OP_MSG_DATA:
                raise BagError(f"{self.path}: chunk at byte {self.chunks[ci].pos}: the index points at a record of op {hdr['op'][0]} "
                               f"at offset {off}, not at a message")
            c = self.connections[conn]
            yield Message(c["topic"], c["type"], t // 1_000_000_000, t % 1_000_000_000, data[start:start + dl])
            if last_use[ci] == i:
                del live[ci]
