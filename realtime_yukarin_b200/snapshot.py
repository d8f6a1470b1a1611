"""The snapshot container (include/ryk.h ryk_snapshot_describe, csrc/snapshot.h; DESIGN.md §4k) on the host side.

A blob is a 32-byte header {magic "RYKSNAP\\0", format version, kind, total bytes, FNV-1a-64 of the bytes after the header} and
tagged sections {four-character tag, 0, payload bytes, payload zero-padded to 8 bytes}, little-endian.  libryk writes session and
re-blocker blobs; `pack` writes the pipeline blob of worker.RealtimePipeline.snapshot, which holds those two and the pipeline's host
state.  `unpack` reads any of them after ryk_snapshot_describe has verified it.
"""
import struct
from typing import Dict, List, Tuple

from .engine import SNAPSHOT_KINDS, describe_snapshot, seal_snapshot

MAGIC = 0x0050414e534b5952
VERSION = 1
KINDS = {v: k for k, v in SNAPSHOT_KINDS.items()}
_HEADER = struct.Struct('<QIIQQ')
_SECTION = struct.Struct('<IIQ')


def _padded(n: int) -> int:
    return (n + 7) & ~7


def pack(kind: str, sections: List[Tuple[str, bytes]], version: int = VERSION) -> bytes:
    """A blob of `kind` ('session', 'reblock' or 'pipeline') holding `sections` [(four-character tag, payload)] in order."""
    body = bytearray()
    for tag, payload in sections:
        t = tag.encode('ascii')
        if len(t) != 4:
            raise ValueError(f'a section tag is four characters: {tag!r}')
        payload = bytes(payload)
        body += _SECTION.pack(int.from_bytes(t, 'little'), 0, len(payload)) + payload + bytes(_padded(len(payload)) - len(payload))
    blob = bytearray(_HEADER.pack(MAGIC, version, KINDS[kind], 0, 0) + bytes(body))
    seal_snapshot(blob)
    return bytes(blob)


def unpack(blob: bytes) -> Tuple[str, Dict[str, bytes]]:
    """(kind, {tag: payload}) of a blob that ryk_snapshot_describe accepts (a tag that repeats keeps its first payload)."""
    blob = bytes(blob)
    d = describe_snapshot(blob)
    out: Dict[str, bytes] = {}
    at = _HEADER.size
    for tag, n in d['sections']:
        at += _SECTION.size
        out.setdefault(tag, blob[at:at + n])
        at += _padded(n)
    return d['kind'], out

