"""Bag writers for what the node publishes: a ROS1 bag (format 2.0) and a rosbag2 recording (sqlite3 storage), with the standard
library only. Both take messages in emission order as write(topic, ROS1 type, (sec, nsec), serialized bytes); the record time is the
stamp given. open_writer picks one by format.

ROS1 (the layout rosbag.py reads): the file header and a bag-header record padded to 4096 bytes; chunks (uncompressed or bz2) that
hold a connection record the first time a connection is used, then message-data records; after every chunk, one index-data record per
connection (record time and offset in the uncompressed chunk of each message). close() appends the connection records and one
chunk-info record per chunk, and rewrites the bag header with their position (index_pos) and counts, so `rosbag` tools can seek the
bag. Every chunk is written whole and flushed (768 KiB of messages, rosbag's default, or one larger message): a run cut short leaves a
bag without an index that rosbag.Bag reads up to its last chunk (and `rosbag reindex` repairs).

rosbag2: <dir>/<name>_0.db3 with the schema, topics and messages tables of the sqlite3 storage, committed every COMMIT_EVERY
messages, and <dir>/metadata.yaml (version 5) written by close(). offered_qos_profiles is left empty. A run cut short leaves the
committed messages and no metadata.yaml (rosbag2.Bag2 does not need it; `ros2 bag reindex` writes it).
"""
from __future__ import annotations

import bz2
import os
import sqlite3
import struct

from . import pubmsg
from .rosbag import MAGIC, OP_BAG_HEADER, OP_CHUNK, OP_CHUNK_INFO, OP_CONNECTION, OP_INDEX_DATA, OP_MSG_DATA, BagError

FORMATS = ("ros1", "ros2")
COMPRESSIONS = ("none", "bz2")


def _fields(d: dict) -> bytes:
    out = b""
    for k, v in d.items():
        f = k.encode() + b"=" + v
        out += struct.pack("<I", len(f)) + f
    return out


def _record(header: dict, data: bytes = b"") -> bytes:
    h = _fields(header)
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def _u32(v):
    return struct.pack("<I", v)


def _time(t):
    return struct.pack("<II", *t)


def _refuse_existing(path):
    if os.path.lexists(path):
        raise BagError(f"{path}: exists; the recording is not written over an existing file or directory")


class Ros1Writer:
    encoding = "ros1"
    CHUNK_BYTES = 768 * 1024
    HEADER_BYTES = 4096

    def __init__(self, path: str, compression: str = "none"):
        if compression not in COMPRESSIONS:
            raise BagError(f"{path}: chunk compression {compression!r}; one of {', '.join(COMPRESSIONS)}")
        _refuse_existing(path)
        self.path, self.compression = path, compression
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        self.f = open(path, "wb")
        self.f.write(MAGIC + self._bag_header(0, 0, 0))
        self.conns = {}         # topic -> (conn id, type)
        self.infos = []         # chunk-info records
        self.chunk = bytearray()
        self.index = {}         # conn id -> [(sec, nsec, offset)] of the open chunk
        self.closed = False

    def _bag_header(self, index_pos, conn_count, chunk_count):
        h = {"op": bytes([OP_BAG_HEADER]), "index_pos": struct.pack("<Q", index_pos), "conn_count": _u32(conn_count),
             "chunk_count": _u32(chunk_count)}
        return _record(h, b" " * (self.HEADER_BYTES - len(_record(h))))

    def _conn_record(self, cid, topic, type_):
        md5, definition = pubmsg.connection(type_)
        body = _fields({"topic": topic.encode(), "type": type_.encode(), "md5sum": md5.encode(),
                        "message_definition": definition.encode()})
        return _record({"op": bytes([OP_CONNECTION]), "conn": _u32(cid), "topic": topic.encode()}, body)

    def write(self, topic: str, type_: str, stamp, data: bytes):
        if topic not in self.conns:
            self.conns[topic] = (len(self.conns), type_)
            self.chunk += self._conn_record(len(self.conns) - 1, topic, type_)
        cid, t = self.conns[topic]
        if t != type_:
            raise BagError(f"{self.path}: topic {topic} written as {type_} and as {t}")
        self.index.setdefault(cid, []).append((*stamp, len(self.chunk)))
        self.chunk += _record({"op": bytes([OP_MSG_DATA]), "conn": _u32(cid), "time": _time(stamp)}, data)
        if len(self.chunk) >= self.CHUNK_BYTES:
            self._flush_chunk()

    def _flush_chunk(self):
        if not self.chunk:
            return
        raw = bytes(self.chunk)
        pos = self.f.tell()
        out = _record({"op": bytes([OP_CHUNK]), "compression": self.compression.encode(), "size": _u32(len(raw))},
                      bz2.compress(raw) if self.compression == "bz2" else raw)
        times = []
        for cid, entries in self.index.items():
            out += _record({"op": bytes([OP_INDEX_DATA]), "ver": _u32(1), "conn": _u32(cid), "count": _u32(len(entries))},
                           b"".join(struct.pack("<III", *e) for e in entries))
            times += [(s, n) for s, n, _ in entries]
        self.f.write(out)
        self.f.flush()
        self.infos.append(_record({"op": bytes([OP_CHUNK_INFO]), "ver": _u32(1), "chunk_pos": struct.pack("<Q", pos),
                                   "start_time": _time(min(times)), "end_time": _time(max(times)), "count": _u32(len(self.index))},
                                  b"".join(struct.pack("<II", cid, len(e)) for cid, e in self.index.items())))
        self.chunk = bytearray()
        self.index = {}

    def close(self):
        if self.closed:
            return
        self.closed = True
        self._flush_chunk()
        index_pos = self.f.tell()
        for topic, (cid, type_) in self.conns.items():
            self.f.write(self._conn_record(cid, topic, type_))
        for r in self.infos:
            self.f.write(r)
        self.f.seek(len(MAGIC))
        self.f.write(self._bag_header(index_pos, len(self.conns), len(self.infos)))
        self.f.close()


SCHEMA = """
CREATE TABLE schema(schema_version INTEGER PRIMARY KEY, ros_distro TEXT NOT NULL);
CREATE TABLE metadata(id INTEGER PRIMARY KEY, metadata_version INTEGER NOT NULL, metadata TEXT NOT NULL);
CREATE TABLE topics(id INTEGER PRIMARY KEY, name TEXT NOT NULL, type TEXT NOT NULL, serialization_format TEXT NOT NULL,
                    offered_qos_profiles TEXT NOT NULL);
CREATE TABLE messages(id INTEGER PRIMARY KEY, topic_id INTEGER NOT NULL, timestamp INTEGER NOT NULL, data BLOB NOT NULL);
CREATE INDEX timestamp_idx ON messages (timestamp ASC);
INSERT INTO schema VALUES (3, 'humble');
"""


class Ros2Writer:
    encoding = "cdr"
    COMMIT_EVERY = 64

    def __init__(self, path: str):
        _refuse_existing(path)
        os.makedirs(path)
        self.path = path
        self.db_name = os.path.basename(os.path.normpath(path)) + "_0.db3"
        self.con = sqlite3.connect(os.path.join(path, self.db_name))
        self.con.executescript(SCHEMA)
        self.topics = {}        # topic -> [topic id, ROS 2 type, count]
        self.pending = 0
        self.t_min = self.t_max = None
        self.closed = False

    def write(self, topic: str, type_: str, stamp, data: bytes):
        t2 = pubmsg.ros2_type(type_)
        if topic not in self.topics:
            self.topics[topic] = [len(self.topics) + 1, t2, 0]
            self.con.execute("INSERT INTO topics VALUES (?, ?, ?, 'cdr', '')", (len(self.topics), topic, t2))
        e = self.topics[topic]
        if e[1] != t2:
            raise BagError(f"{self.path}: topic {topic} written as {t2} and as {e[1]}")
        ns = stamp[0] * 1_000_000_000 + stamp[1]
        self.con.execute("INSERT INTO messages(topic_id, timestamp, data) VALUES (?, ?, ?)", (e[0], ns, data))
        e[2] += 1
        self.t_min = ns if self.t_min is None else min(self.t_min, ns)
        self.t_max = ns if self.t_max is None else max(self.t_max, ns)
        self.pending += 1
        if self.pending >= self.COMMIT_EVERY:
            self.con.commit()
            self.pending = 0

    def metadata(self) -> str:
        n = sum(e[2] for e in self.topics.values())
        t0 = self.t_min or 0
        dur = (self.t_max - self.t_min) if self.t_min is not None else 0
        topics = "".join(f"    - topic_metadata:\n        name: {topic}\n        type: {t2}\n        serialization_format: cdr\n"
                         f"        offered_qos_profiles: \"\"\n      message_count: {cnt}\n" for topic, (_, t2, cnt) in self.topics.items())
        return ("rosbag2_bagfile_information:\n  version: 5\n  storage_identifier: sqlite3\n"
                f"  duration:\n    nanoseconds: {dur}\n  starting_time:\n    nanoseconds_since_epoch: {t0}\n  message_count: {n}\n"
                "  topics_with_message_count:" + ("\n" + topics if topics else " []\n")
                + "  compression_format: \"\"\n  compression_mode: \"\"\n"
                f"  relative_file_paths:\n    - {self.db_name}\n"
                f"  files:\n    - path: {self.db_name}\n      starting_time:\n        nanoseconds_since_epoch: {t0}\n"
                f"      duration:\n        nanoseconds: {dur}\n      message_count: {n}\n")

    def close(self):
        if self.closed:
            return
        self.closed = True
        self.con.commit()
        self.con.close()
        with open(os.path.join(self.path, "metadata.yaml"), "w") as f:
            f.write(self.metadata())


def open_writer(path: str, fmt: str, compression: str = "none"):
    """A Ros1Writer (fmt "ros1", compression "none" or "bz2") or a Ros2Writer (fmt "ros2", uncompressed) at path, which must not
    exist."""
    if fmt == "ros1":
        return Ros1Writer(path, compression)
    if fmt == "ros2":
        if compression != "none":
            raise BagError(f"{path}: --record-compression {compression} applies to ROS1 bags; a rosbag2 recording is written uncompressed")
        return Ros2Writer(path)
    raise BagError(f"{path}: unknown recording format {fmt!r}; one of {', '.join(FORMATS)}")
