"""A rosbag2 reader for the sqlite3 storage: the messages of chosen topics of a ROS 2 recording in timestamp order, with the standard
library's sqlite3 and numpy only.

A recording is a directory with metadata.yaml and one or more <name>_<N>.db3 files (a recording split by size or duration has
several); a single .db3 file can also be read on its own. Every .db3 holds

    topics(id, name, type, serialization_format, ...)   the columns that newer distributions add are ignored
    messages(id, topic_id, timestamp, data)             timestamp: receive time [ns]; data: the CDR bytes (rosmsg's *_cdr decoders)

metadata.yaml is not read: every *.db3 of the directory is.

A finished recording is opened read-only and `immutable`: no lock and no journal, so it also opens from read-only media. A .db3 with a
non-empty write-ahead log beside it (<file>.db3-wal: a WAL-mode recording, e.g. rosbag2's `resilient` preset, whose recorder died
before it checkpointed) keeps its newest messages, or even its tables, only in that log. Such a file is opened read-only without
`immutable`, so that SQLite replays the log, with a BagWarning; SQLite then needs to create <file>.db3-shm next to it, and where it
cannot, the file is refused with a BagError that names the log.

Delivery (decision): ascending timestamp across all files; ties go by file, in the numeric order of its _N suffix, then by
messages.id. This is the analogue of the ROS1 reader's (record time, file position) order. Each file is streamed through an ordered
cursor and the streams are merged (heapq.merge); no file is loaded whole.

Refused with a BagError that says what was found and where: a chosen topic whose serialization_format is not cdr, a message that
starts with a zstd frame (per-message compression), a *.db3.zstd file (per-file compression), an MCAP file, big-endian CDR, a
directory without a .db3 file, and a damaged database (an SQLite error while it is read).
"""
from __future__ import annotations

import contextlib
import heapq
import os
import pathlib
import re
import sqlite3
import warnings

from . import rosbag
from .rosbag import BagError, BagWarning, Message

SQLITE_MAGIC = b"SQLite format 3\0"
MCAP_MAGIC = b"\x89MCAP0\r\n"
ZSTD_MAGIC = b"\x28\xb5\x2f\xfd"


def _head(path: str, n: int = 16) -> bytes:
    with open(path, "rb") as f:
        return f.read(n)


def _file_order(name: str):
    """Split files in the numeric order of their _N suffix (rec_2.db3 before rec_10.db3)."""
    m = re.search(r"_(\d+)\.db3$", name)
    return (int(m.group(1)) if m else -1, name)


def _refuse_compressed(path: str):
    raise BagError(f"{path}: a rosbag2 file compressed with zstd (compression_mode FILE); compressed recordings are not read. "
                   f"Record without --compression-mode, or convert the recording to an uncompressed sqlite3 one")


def _refuse_mcap(path: str):
    raise BagError(f"{path}: an MCAP file; only the sqlite3 storage of rosbag2 (.db3) is read")


@contextlib.contextmanager
def _read_errors(p: str):
    """A damaged database (an SQLite error while reading it) is a BagError that names the file."""
    try:
        yield
    except sqlite3.DatabaseError as e:
        raise BagError(f"{p}: reading the database failed ({e}); the file is damaged") from None


def _stream(cur, fi, p):
    with _read_errors(p):
        for ts, mid, tid, data in cur:
            yield ts, fi, mid, tid, data


class Bag2:
    """bag = Bag2(dir or file.db3); the interface of rosbag.Bag: bag.topics() -> {topic: type}; bag.check_topics(wanted);
    bag.count(wanted); for m in bag.messages({topic: (type, ...)}): ... (rosbag.Message, sec / nsec from the timestamp)."""
    format = "cdr"      # the serialization of its messages (rosmsg.decoders)

    def __init__(self, path: str):
        self.path = path
        self.files = []     # [(file path, sqlite3 connection, {topic id: (name, type, serialization_format)})] in delivery order
        if os.path.isdir(path):
            names = sorted(os.listdir(path))
            for n in names:
                if n.endswith(".db3.zstd"):
                    _refuse_compressed(os.path.join(path, n))
            dbs = sorted((n for n in names if n.endswith(".db3")), key=_file_order)
            if not dbs:
                mcap = [n for n in names if n.endswith(".mcap")]
                if mcap:
                    _refuse_mcap(os.path.join(path, mcap[0]))
                raise BagError(f"{path}: a directory without a .db3 file; it holds: {', '.join(names) or '(nothing)'}")
            paths = [os.path.join(path, n) for n in dbs]
        else:
            paths = [path]
        try:
            for p in paths:
                self._open(p)
        except BaseException:
            self.close()
            raise

    def _open(self, p: str):
        head = _head(p)
        if head.startswith(MCAP_MAGIC):
            _refuse_mcap(p)
        if head.startswith(ZSTD_MAGIC) or p.endswith(".zstd"):
            _refuse_compressed(p)
        if not head.startswith(SQLITE_MAGIC):
            raise BagError(f"{p}: not a rosbag2 sqlite3 file (it starts with {head!r})")
        wal = p + "-wal"
        live_wal = os.path.isfile(wal) and os.path.getsize(wal) > 0
        if live_wal:
            warnings.warn(f"{wal}: the recording's newest messages are still in its write-ahead log (a recorder that did not close it?); "
                          f"SQLite replays the log and they are read too", BagWarning, stacklevel=4)
        con = sqlite3.connect(pathlib.Path(p).resolve().as_uri() + ("?mode=ro" if live_wal else "?mode=ro&immutable=1"), uri=True)
        self.files.append((p, con, {}))
        try:
            rows = con.execute("SELECT id, name, type, serialization_format FROM topics").fetchall()
            con.execute("SELECT id, topic_id, timestamp, data FROM messages LIMIT 0")
        except sqlite3.DatabaseError as e:
            if live_wal and isinstance(e, sqlite3.OperationalError) and "no such table" not in str(e):
                raise BagError(f"{p}: its write-ahead log {wal} holds messages that were never checkpointed, and SQLite cannot replay it "
                               f"here ({e}); copy the recording to a writable directory and read it there") from None
            raise BagError(f"{p}: not a rosbag2 database ({e})") from None
        self.files[-1][2].update((tid, (name, type_, fmt)) for tid, name, type_, fmt in rows)

    def close(self):
        for _, con, _ in self.files:
            con.close()
        self.files = []

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- the interface of rosbag.Bag ----
    def topics(self) -> dict:
        """{topic: message type} of every file's topics."""
        return {name: type_ for _, _, t in self.files for name, type_, _ in t.values()}

    def _describe(self) -> str:
        t = self.topics()
        return "; ".join(f"{k} [{v}]" for k, v in sorted(t.items())) or "(none)"

    def check_topics(self, wanted: dict) -> dict:
        """wanted {topic: accepted type or tuple of types}. Raises BagError naming the bag's topics for a missing topic or a topic of
        another type, and for a chosen topic that is not serialized as cdr. Returns {file index: {topic id: topic}}."""
        out = {fi: {} for fi in range(len(self.files))}
        for topic, types in wanted.items():
            types = (types,) if isinstance(types, str) else tuple(types)
            found = False
            for fi, (p, _, t) in enumerate(self.files):
                for tid, (name, type_, fmt) in t.items():
                    if name != topic:
                        continue
                    found = True
                    if type_ not in types:
                        raise BagError(f"{self.path}: topic {topic!r} carries {type_}, expected {' or '.join(types)}; the bag has: "
                                       f"{self._describe()}")
                    if fmt != "cdr":
                        raise BagError(f"{p}: topic {topic!r} is serialized as {fmt!r}; only cdr is read")
                    out[fi][tid] = topic
            if not found:
                raise BagError(f"{self.path}: no topic {topic!r} in the bag; it has: {self._describe()}")
        return out

    def _select(self, chosen: dict, cols: str, tail: str = ""):
        """(file index, file path, cursor) of `SELECT cols FROM messages` over the chosen topics of every file that has one."""
        for fi, ids in chosen.items():
            if ids:
                p, con, _ = self.files[fi]
                marks = ",".join("?" * len(ids))
                with _read_errors(p):
                    cur = con.execute(f"SELECT {cols} FROM messages WHERE topic_id IN ({marks}){tail}", sorted(ids))
                yield fi, p, cur

    def count(self, wanted: dict) -> int:
        n = 0
        for _, p, cur in self._select(self.check_topics(wanted), "COUNT(*)"):
            with _read_errors(p):
                n += cur.fetchone()[0]
        return n

    def time_bounds(self):
        """(first, last) timestamp [ns] of all messages, or None for a bag without messages."""
        b = []
        for p, con, _ in self.files:
            with _read_errors(p):
                b.append(con.execute("SELECT MIN(timestamp), MAX(timestamp) FROM messages").fetchone())
        b = [x for x in b if x[0] is not None]
        return (min(x[0] for x in b), max(x[1] for x in b)) if b else None

    def messages(self, wanted: dict):
        """Yield the Message of every message of the chosen topics in (timestamp, file, id) order."""
        chosen = self.check_topics(wanted)
        streams = [_stream(cur, fi, p) for fi, p, cur in self._select(chosen, "timestamp, id, topic_id, data", " ORDER BY timestamp, id")]
        for ts, fi, mid, tid, data in heapq.merge(*streams):
            p, _, t = self.files[fi]
            name, type_, _ = t[tid]
            head = bytes(data[:4])
            if head == ZSTD_MAGIC:
                raise BagError(f"{p}: message {mid} on {name} starts with a zstd frame (compression_mode MESSAGE); compressed "
                               f"recordings are not read")
            if head[:2] == b"\0\0":
                raise BagError(f"{p}: message {mid} on {name} is big-endian CDR (encapsulation {head.hex(' ')}); only little-endian "
                               f"CDR is read")
            yield Message(name, type_, ts // 1_000_000_000, ts % 1_000_000_000, data)


def open_bag(path: str):
    """A ROS1 bag (rosbag.Bag), a rosbag2 directory or a rosbag2 .db3 file (Bag2), told apart by whether the path is a directory and
    by the file's first bytes, not by its extension. MCAP and zstd-compressed files are refused by name."""
    if os.path.isdir(path):
        return Bag2(path)
    head = _head(path)
    if head.startswith(b"#ROSBAG"):
        return rosbag.Bag(path)
    if head.startswith((SQLITE_MAGIC, MCAP_MAGIC, ZSTD_MAGIC)):
        return Bag2(path)
    raise BagError(f"{path}: neither a ROS1 bag, a rosbag2 directory nor a rosbag2 .db3 file (it starts with {head!r})")
