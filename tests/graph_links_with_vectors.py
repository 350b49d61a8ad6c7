"""Restatement of the reference's HNSW links format with inline vectors (GraphLinksFormat::CompressedWithVectors), for tests and
tools (test infrastructure, never imported by the product).

Writer: serialize_graph_links for GraphLinksFormatParam::CompressedWithVectors (lib/segment/src/index/hnsw_index/graph_links/
serializer.rs:32-49, 91-171, 223-238): header (header.rs:37-70), level offsets, reindex, zero padding to a file offset that is a
multiple of max(base align, link align), the records, the compressed byte offsets.  A record is
[base vector, level 0 only][varint link count][packed links][pad to link align][count x link vector][level 0: pad to base align].

Reader: GraphLinksView::load_compressed_with_vectors / links_with_vectors / point_level (view.rs:165-207, 276-369), value by value.
The bit-level pieces (pack_links, iterate_packed_links, packed_links_size, bitpacking_ordered) are those of
tests/graph_links_compressed.py.
"""
from __future__ import annotations

import numpy as np

from tests import graph_links_compressed as gl

HEADER_SIZE = 80


def write_varint(v: int) -> bytes:
    """integer_encoding VarInt (LEB128) of a u64"""
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def decode_varint(data: bytes, pos: int, end: int):
    """u64::decode_var(&data[pos..end]): (value, size) or None"""
    v = 0
    for i in range(10):
        if pos + i >= end:
            return None
        b = data[pos + i]
        v |= (b & 0x7F) << (7 * i)
        if not b & 0x80:
            return v, i + 1
    return None


def _next_multiple(x: int, a: int) -> int:
    return -(-x // a) * a


def serialize_with_vectors(edges, m: int, m0: int, base_vector, link_vector, base_layout, link_layout, chunk_len_log2: int | None = None) -> bytes:
    """serialize_graph_links(edges, CompressedWithVectors, HnswM { m, m0 }).  base_vector(id) / link_vector(id) -> bytes;
    base_layout / link_layout = (size, align)."""
    (bsize, balign), (lsize, lalign) = base_layout, link_layout
    assert bsize % balign == 0 and lsize % lalign == 0, "vector size must be a multiple of its alignment"
    n = len(edges)
    lo, reindex, _, _ = gl.edges_to_plain_arrays(edges)
    nlev = np.array([len(e) for e in edges], dtype=np.int64)
    back = np.argsort(-nlev, kind="stable")
    levels = int(nlev.max()) if n else 0
    bpu = gl.bits_per_unsorted(n)
    pos = HEADER_SIZE + 8 * len(lo) + 4 * n
    pad = _next_multiple(pos, max(balign, lalign)) - pos
    rec = bytearray()
    offsets = [0]
    for level in range(levels):
        count = int((nlev > level).sum())
        ids = range(count) if level == 0 else back[:count]
        level_m = m0 if level == 0 else m
        for i in ids:
            i = int(i)
            if level == 0:
                b = bytes(base_vector(i))
                assert len(b) == bsize, "vector size mismatch"
                rec += b
            raw = edges[i][level]
            rec += write_varint(len(raw))
            packed, stored = gl.pack_links(raw, bpu, level_m)
            rec += packed
            rec += b"\0" * (_next_multiple(len(rec), lalign) - len(rec))
            for x in stored:
                v = bytes(link_vector(int(x)))
                assert len(v) == lsize, "vector size mismatch"
                rec += v
            if level == 0:
                rec += b"\0" * (_next_multiple(len(rec), balign) - len(rec))
            offsets.append(len(rec))
    coff, p = gl.compress(offsets, chunk_len_log2)
    hdr = bytearray(HEADER_SIZE)
    hdr[0:8] = n.to_bytes(8, "little")
    hdr[8:16] = gl.VERSION_COMPRESSED_WITH_VECTORS.to_bytes(8, "little")
    hdr[16:24] = len(lo).to_bytes(8, "little")
    hdr[24:32] = len(rec).to_bytes(8, "little")
    hdr[32:40] = p.length.to_bytes(8, "little")
    hdr[40], hdr[41], hdr[42] = p.base_bits, p.delta_bits, p.chunk_len_log2
    hdr[43:51] = int(m).to_bytes(8, "little")
    hdr[51:59] = int(m0).to_bytes(8, "little")
    hdr[59:67] = int(bsize).to_bytes(8, "little")
    hdr[67] = balign
    hdr[68:76] = int(lsize).to_bytes(8, "little")
    hdr[76] = lalign
    return b"".join([bytes(hdr), np.asarray(lo, np.uint64).tobytes(), reindex.tobytes(), b"\0" * pad, bytes(rec), coff])


class WithVectorsLinks:
    """GraphLinksView::load_compressed_with_vectors + links_with_vectors() + point_level(), value by value."""

    def __init__(self, blob):
        b = bytes(blob) if isinstance(blob, (bytes, bytearray)) else bytes(np.ascontiguousarray(blob, dtype=np.uint8).tobytes())
        u = lambda o: int.from_bytes(b[o:o + 8], "little")
        self.point_count, self.version, self.levels_count, self.total_neighbors_bytes = u(0), u(8), u(16), u(24)
        assert self.version == gl.VERSION_COMPRESSED_WITH_VECTORS
        self.params = gl.Parameters(u(32), b[40], b[41], b[42])
        self.m, self.m0 = u(43), u(51)
        self.base_size, self.base_align, self.link_size, self.link_align = u(59), b[67], u(68), b[76]
        assert self.params.valid() and self.link_size > 0
        p = HEADER_SIZE
        self.level_offsets = [u(p + 8 * i) for i in range(self.levels_count)] + [self.params.length - 1]
        p += 8 * self.levels_count
        self.reindex = np.frombuffer(b, dtype=np.uint32, count=self.point_count, offset=p)
        p += 4 * self.point_count
        p = _next_multiple(p, max(self.base_align, self.link_align))
        self.records_at = p
        self.neighbors = b[p:p + self.total_neighbors_bytes]
        assert len(self.neighbors) == self.total_neighbors_bytes
        p += self.total_neighbors_bytes
        self.offsets = b[p:p + self.params.compressed_size_bytes()]
        assert len(self.offsets) == self.params.compressed_size_bytes()
        self.bits_per_unsorted = gl.bits_per_unsorted(self.point_count)

    def level_m(self, level: int) -> int:
        return self.m0 if level == 0 else self.m

    def point_level(self, point: int) -> int:
        r = int(self.reindex[point])
        lo = self.level_offsets
        for level in range(len(lo) - 2):
            if r >= lo[level + 2] - lo[level + 1]:
                return level
        return len(lo) - 2

    def record(self, point: int, level: int):
        """(base vector bytes, links, link vector bytes per link, byte offset of the first link vector in the records)"""
        idx = point if level == 0 else self.level_offsets[level] + int(self.reindex[point])
        start, end = gl.read_pair(self.offsets, self.params, idx)
        nb = self.neighbors
        pos = start
        base = b""
        if level == 0:
            base = nb[pos:pos + self.base_size]
            pos += self.base_size
        count, size = decode_varint(nb, pos, end)
        pos += size
        lsize = gl.packed_links_size(nb[pos:end], self.bits_per_unsorted, self.level_m(level), count)
        links = gl.iterate_packed_links(nb[pos:pos + lsize], self.bits_per_unsorted, self.level_m(level))
        pos = _next_multiple(pos + lsize, self.link_align)
        vecs = [nb[pos + i * self.link_size:pos + (i + 1) * self.link_size] for i in range(count)]
        assert len(links) == count and all(len(v) == self.link_size for v in vecs)
        return base, links, vecs, pos

    def links_with_vectors(self, point: int, level: int):
        base, links, vecs, _ = self.record(point, level)
        return base, links, vecs

    def links(self, point: int, level: int) -> list[int]:
        return self.record(point, level)[1]

    def to_edges(self):
        return [[self.links(p, lvl) for lvl in range(self.point_level(p) + 1)] for p in range(self.point_count)]


def edges_of_plain(blob):
    """edges[point][level] of a plain links.bin (the oracle's and the device's export), in stored order"""
    n, lo, reindex, nb, off = gl.parse_plain(blob)
    lo = [int(x) for x in lo] + [len(off) - 1]
    levels = len(lo) - 1
    edges = []
    for p in range(n):
        r = int(reindex[p])
        lv = []
        for lvl in range(levels):
            if lvl > 0 and r >= lo[lvl + 1] - lo[lvl]:
                break
            idx = p if lvl == 0 else lo[lvl] + r
            lv.append([int(x) for x in nb[int(off[idx]):int(off[idx + 1])]])
        edges.append(lv)
    return edges


def serialize_plain_with_vectors(blob, m: int, m0: int, base_rows: np.ndarray, link_rows: np.ndarray) -> np.ndarray:
    """CompressedWithVectors of the graph a plain links.bin holds (same reindex), with f32 base vectors (base_rows: [n, dim * 4] u8,
    alignment 4) and link vectors of alignment 1 (link_rows: [n, L] u8, the SQ8 row layout), for graphs of millions of points: the
    links are packed in batches with numpy (_pack_entries) and each record is copied in place.  Returns the file as a uint8 array."""
    n, lo, reindex, nb, off = gl.parse_plain(blob)
    bsize, lsize = base_rows.shape[1], link_rows.shape[1]
    assert bsize % 4 == 0
    bpu = gl.bits_per_unsorted(n)
    n_e = off.size - 1
    cnt = np.diff(off).astype(np.int64)
    assert cnt.max(initial=0) < 1 << 14
    sc = np.where(np.arange(n_e) < n, m0, m).astype(np.int64)
    packed, psize = gl._pack_entries(nb, off - off[0], sc, bpu)
    packed = np.frombuffer(packed, np.uint8)
    pstart = np.r_[0, np.cumsum(psize)[:-1]]
    # stored order: the first min(count, level_m) links sorted, the rest as given (pack_links)
    ent = np.repeat(np.arange(n_e), cnt)
    k = np.arange(nb.size) - np.repeat(off[:-1].astype(np.int64), cnt)
    ns = np.minimum(cnt, sc)
    tail = k >= ns[ent]
    order = np.lexsort((np.where(tail, k, nb.astype(np.int64)), tail, ent))
    stored = nb[order]
    vsz = np.where(cnt < 128, 1, 2)
    # level-0 records start at a multiple of 4 and are padded to one, links need no alignment: sizes do not depend on positions
    size = vsz + psize + cnt * lsize
    size[:n] += bsize
    size[:n] = (size[:n] + 3) // 4 * 4
    rstart = np.r_[0, np.cumsum(size)[:-1]]
    total = int(size.sum())
    boff = np.r_[rstart, total].astype(np.uint64)
    coff, p = gl.compress(boff)
    head = HEADER_SIZE + 8 * lo.size + 4 * n
    pad = _next_multiple(head, 4) - head
    out = np.zeros(head + pad + total + len(coff), np.uint8)
    hdr = out[:HEADER_SIZE]
    hdr[0:8] = np.frombuffer(int(n).to_bytes(8, "little"), np.uint8)
    hdr[8:16] = np.frombuffer(gl.VERSION_COMPRESSED_WITH_VECTORS.to_bytes(8, "little"), np.uint8)
    hdr[16:24] = np.frombuffer(int(lo.size).to_bytes(8, "little"), np.uint8)
    hdr[24:32] = np.frombuffer(total.to_bytes(8, "little"), np.uint8)
    hdr[32:40] = np.frombuffer(p.length.to_bytes(8, "little"), np.uint8)
    hdr[40], hdr[41], hdr[42] = p.base_bits, p.delta_bits, p.chunk_len_log2
    hdr[43:51] = np.frombuffer(int(m).to_bytes(8, "little"), np.uint8)
    hdr[51:59] = np.frombuffer(int(m0).to_bytes(8, "little"), np.uint8)
    hdr[59:67] = np.frombuffer(int(bsize).to_bytes(8, "little"), np.uint8)
    hdr[67] = 4
    hdr[68:76] = np.frombuffer(int(lsize).to_bytes(8, "little"), np.uint8)
    hdr[76] = 1
    out[HEADER_SIZE:HEADER_SIZE + 8 * lo.size] = np.asarray(lo, np.uint64).view(np.uint8)
    out[HEADER_SIZE + 8 * lo.size:head] = np.asarray(reindex, np.uint32).view(np.uint8)
    rec = out[head + pad:head + pad + total]
    out[head + pad + total:] = np.frombuffer(coff, np.uint8)
    for e in range(n_e):
        a = int(rstart[e])
        if e < n:
            rec[a:a + bsize] = base_rows[e]
            a += bsize
        c = int(cnt[e])
        if c < 128:
            rec[a] = c; a += 1
        else:
            rec[a] = (c & 127) | 128; rec[a + 1] = c >> 7; a += 2
        ps = int(psize[e])
        rec[a:a + ps] = packed[int(pstart[e]):int(pstart[e]) + ps]
        a += ps
        if c:
            rec[a:a + c * lsize] = link_rows[stored[int(off[e]):int(off[e + 1])]].reshape(-1)
    return out
