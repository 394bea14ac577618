#!/usr/bin/env python
"""Minimal pure-Python reader for USDC ("PXR-USDC" crate) files -- just enough to pull array attributes such as a Mesh's
`points` / `faceVertexIndices` out of the reference's binary assets without `pxr` (not installed here).
Format notes: SURVEY.md Appendix C.  Used on the reference's assets, which are not part of this repository.
"""
from __future__ import annotations

import struct

import numpy as np


def lz4_block_decode(src: bytes, out_size: int) -> bytes:
    out = bytearray()
    i, n = 0, len(src)
    while i < n:
        tok = src[i]; i += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = src[i]; i += 1
                lit += b
                if b != 255:
                    break
        out += src[i:i + lit]; i += lit
        if i >= n:
            break
        off = src[i] | (src[i + 1] << 8); i += 2
        ml = tok & 15
        if ml == 15:
            while True:
                b = src[i]; i += 1
                ml += b
                if b != 255:
                    break
        ml += 4
        start = len(out) - off
        if off >= ml:
            out += out[start:start + ml]
        else:
            for k in range(ml):
                out.append(out[start + k])
    assert len(out) == out_size, (len(out), out_size)
    return bytes(out)


def fast_decompress(buf: bytes, out_size: int) -> bytes:
    """TfFastCompression: first byte = number of chunks (0 => the rest is ONE raw LZ4 block)."""
    nchunks = buf[0]
    if nchunks == 0:
        return lz4_block_decode(buf[1:], out_size)
    out, pos = bytearray(), 1
    for _ in range(nchunks):
        (csz,) = struct.unpack_from("<i", buf, pos); pos += 4
        remaining = out_size - len(out)
        out += lz4_block_decode(buf[pos:pos + csz], min(remaining, 127 * 1024 * 1024)) if False else b""
        pos += csz
    raise NotImplementedError("multi-chunk fast compression")


def decode_ints(buf: bytes, n: int, width: int = 4) -> np.ndarray:
    """USD integer coding (after LZ4): int common; 2-bit codes per value (0 common, 1 int8, 2 int16, 3 int32 delta);
    values are running sums."""
    (common,) = struct.unpack_from("<i", buf, 0)
    ncode_bytes = (n * 2 + 7) // 8
    codes_raw = np.frombuffer(buf, dtype=np.uint8, count=ncode_bytes, offset=4)
    codes = np.empty(ncode_bytes * 4, dtype=np.uint8)
    for k in range(4):
        codes[k::4] = (codes_raw >> (2 * k)) & 3
    codes = codes[:n]
    sizes = np.array([0, 1, 2, 4], dtype=np.int64)[codes]
    offs = 4 + ncode_bytes + np.concatenate([[0], np.cumsum(sizes)[:-1]])
    data = np.frombuffer(buf, dtype=np.uint8)
    deltas = np.full(n, common, dtype=np.int64)
    m1 = codes == 1
    deltas[m1] = data[offs[m1]].view(np.int8)
    m2 = codes == 2
    if m2.any():
        o = offs[m2]
        deltas[m2] = (data[o].astype(np.int64) | (data[o + 1].astype(np.int64) << 8)).astype(np.uint16).view(np.int16)
    m3 = codes == 3
    if m3.any():
        o = offs[m3]
        v = (data[o].astype(np.int64) | (data[o + 1].astype(np.int64) << 8) | (data[o + 2].astype(np.int64) << 16) | (data[o + 3].astype(np.int64) << 24))
        deltas[m3] = v.astype(np.uint32).view(np.int32)
    return np.cumsum(deltas)


def read_compressed_ints(f: bytes, pos: int, n: int):
    (csz,) = struct.unpack_from("<Q", f, pos); pos += 8
    raw_size = 4 + (n * 2 + 7) // 8 + n * 4            # upper bound of the encoded buffer
    enc = fast_decompress_unknown(f[pos:pos + csz], raw_size)
    return decode_ints(enc, n), pos + csz


def fast_decompress_unknown(buf: bytes, max_size: int) -> bytes:
    """LZ4 block whose exact output size is not stored: decode until the input is exhausted."""
    assert buf[0] == 0, "multi-chunk not supported"
    src = buf[1:]
    out = bytearray()
    i, n = 0, len(src)
    while i < n:
        tok = src[i]; i += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = src[i]; i += 1
                lit += b
                if b != 255:
                    break
        out += src[i:i + lit]; i += lit
        if i >= n:
            break
        off = src[i] | (src[i + 1] << 8); i += 2
        ml = tok & 15
        if ml == 15:
            while True:
                b = src[i]; i += 1
                ml += b
                if b != 255:
                    break
        ml += 4
        start = len(out) - off
        if off >= ml:
            out += out[start:start + ml]
        else:
            for k in range(ml):
                out.append(out[start + k])
    return bytes(out)


class Crate:
    def __init__(self, path: str):
        self.f = open(path, "rb").read()
        f = self.f
        assert f[:8] == b"PXR-USDC", "not a USDC crate"
        self.version = tuple(f[8:11])
        (toc,) = struct.unpack_from("<q", f, 16)
        (nsec,) = struct.unpack_from("<Q", f, toc)
        self.sections = {}
        for k in range(nsec):
            name, start, size = struct.unpack_from("<16sqq", f, toc + 8 + 32 * k)
            self.sections[name.rstrip(b"\0").decode()] = (start, size)
        self._tokens()
        self._fields()

    def _tokens(self):
        start, _ = self.sections["TOKENS"]
        n, usize, csize = struct.unpack_from("<QQQ", self.f, start)
        raw = fast_decompress_unknown(self.f[start + 24:start + 24 + csize], usize)
        self.tokens = [t.decode("utf8", "replace") for t in raw.split(b"\0")[:n]]

    def _fields(self):
        start, _ = self.sections["FIELDS"]
        (n,) = struct.unpack_from("<Q", self.f, start)
        tok_idx, pos = read_compressed_ints(self.f, start + 8, n)
        (csz,) = struct.unpack_from("<Q", self.f, pos); pos += 8
        reps = np.frombuffer(fast_decompress_unknown(self.f[pos:pos + csz], n * 8), dtype="<u8", count=n)
        self.fields = [(self.tokens[int(t)], int(r)) for t, r in zip(tok_idx, reps)]

    def array_fields(self, name: str):
        """All value-reps of fields called `name` that are (non-inlined) arrays: [(type, compressed, offset)]."""
        out = []
        for tok, rep in self.fields:
            if tok != name:
                continue
            is_array, inlined, compressed = (rep >> 63) & 1, (rep >> 62) & 1, (rep >> 61) & 1
            ty = (rep >> 48) & 0xFF
            if is_array and not inlined:
                out.append((ty, bool(compressed), rep & ((1 << 48) - 1)))
        return out

    def read_vec3f_array(self, offset: int) -> np.ndarray:
        (n,) = struct.unpack_from("<Q", self.f, offset)
        return np.frombuffer(self.f, dtype="<f4", count=3 * n, offset=offset + 8).reshape(n, 3).copy()

    def read_int_array(self, offset: int, compressed: bool) -> np.ndarray:
        (n,) = struct.unpack_from("<Q", self.f, offset)
        if not compressed:
            return np.frombuffer(self.f, dtype="<i4", count=n, offset=offset + 8).astype(np.int64)
        vals, _ = read_compressed_ints(self.f, offset + 8, n)
        return vals


if __name__ == "__main__":
    import sys
    c = Crate(sys.argv[1])
    print("version", c.version, "sections", {k: v for k, v in c.sections.items()})
    for name in ("points", "faceVertexCounts", "faceVertexIndices", "extent"):
        print(name, c.array_fields(name)[:4])
