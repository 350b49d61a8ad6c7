"""Restatement of the reference's compressed HNSW links format, for tests and tools (test infrastructure, never imported by
the product).

Writer: serialize_graph_links for GraphLinksFormatParam::Compressed (lib/segment/src/index/hnsw_index/graph_links/
serializer.rs:44-194) with pack_links (common/src/bitpacking_links.rs:23-63) and bitpacking_ordered::compress (including
Parameters::find_best, bitpacking_ordered.rs:196-228); `chunk_len_log2` can be forced so tests reach every parameter set.
The graph writer packs whole batches of entries with numpy, so 10M-point graphs take seconds, not hours.

Reader: an independent per-value restatement of BitReader (bitpacking.rs:84-160), iterate_packed_links
(bitpacking_links.rs:65-133), SliceReader::read_pair (bitpacking_ordered.rs:108-125) and GraphLinksView::load_compressed /
links / point_level (graph_links/view.rs:137-163, 209-263, 354-369).

Nothing here is pinned to bytes the reference wrote (its Rust cannot be built here): format parity is pinned by the
re-typed reference tests in tests/test_graph_links_compressed.py.
"""
from __future__ import annotations

import numpy as np

VERSION_COMPRESSED = 0xFFFF_FFFF_FFFF_FF01
VERSION_COMPRESSED_WITH_VECTORS = 0xFFFF_FFFF_FFFF_FF02
MIN_BITS_PER_VALUE = 8
HEADER_BITS = 5
MAX_CHUNK_LEN_LOG2 = 7
TAIL_SIZE = 7
M64 = (1 << 64) - 1


def packed_bits(v: int) -> int:
    return int(v).bit_length()


def make_bitmask(bits: int) -> int:
    return M64 if bits >= 64 else (1 << bits) - 1


# ------------------------------------------------------------------------------------------------ bit I/O, LSB first
class BitWriter:
    """bitpacking.rs:14-58 (u64 buffer, flushed little-endian; finish() writes the partly filled bytes)."""

    def __init__(self, out: bytearray):
        self.out, self.buf, self.buf_bits = out, 0, 0

    def write(self, value: int, bits: int) -> None:
        assert packed_bits(value) <= bits <= 64
        self.buf |= (value << self.buf_bits) & M64
        self.buf_bits += bits
        if self.buf_bits >= 64:
            self.out += self.buf.to_bytes(8, "little")
            self.buf_bits -= 64
            self.buf = 0 if bits - self.buf_bits == 64 else value >> (bits - self.buf_bits)

    def finish(self) -> None:
        self.out += self.buf.to_bytes(8, "little")[: (self.buf_bits + 7) // 8]


class BitReader:
    """bitpacking.rs:84-160: reads `bits`-wide values; past the end of the input it reads zero bytes."""

    def __init__(self, data: bytes):
        self.data, self.pos, self.buf, self.buf_bits, self.bits, self.mask = bytes(data), 0, 0, 0, 0, 0

    def set_bits(self, bits: int) -> None:
        self.bits, self.mask = bits, make_bitmask(bits)

    def read(self) -> int:
        if self.buf_bits >= self.bits:
            self.buf_bits -= self.bits
            val = self.buf & self.mask
            self.buf >>= self.bits
            return val
        new = int.from_bytes(self.data[self.pos:self.pos + 8].ljust(8, b"\0"), "little")
        self.pos += 8
        val = (self.buf | ((new << self.buf_bits) & M64)) & self.mask
        self.buf_bits += 64 - self.bits
        self.buf = 0 if self.buf_bits == 0 else new >> (64 - self.buf_bits)
        return val


# ------------------------------------------------------------------------------------------------ links of one node
def pack_links(raw_links, bits_per_unsorted: int, sorted_count: int) -> tuple[bytes, list[int]]:
    """bitpacking_links.rs:23-63: (packed bytes, the links in stored order = first min(len, sorted_count) sorted)."""
    links = [int(x) for x in raw_links]
    if not links:
        return b"", []
    ns = min(len(links), sorted_count)
    links[:ns] = sorted(links[:ns])
    out = bytearray()
    w = BitWriter(out)
    if ns:
        deltas = [links[0]] + [links[i] - links[i - 1] for i in range(1, ns)]
        bps = max(packed_bits(max(deltas)), MIN_BITS_PER_VALUE)
        w.write(bps - MIN_BITS_PER_VALUE, HEADER_BITS)
        for d in deltas:
            w.write(d, bps)
    for v in links[ns:]:
        w.write(v, bits_per_unsorted)
    w.finish()
    return bytes(out), links


def iterate_packed_links(data: bytes, bits_per_unsorted: int, sorted_count: int) -> list[int]:
    """bitpacking_links.rs:65-133 (PackedLinksIterator::next)."""
    r = BitReader(data)
    remaining = len(data) * 8
    target = remaining
    if sorted_count != 0 and len(data):
        r.set_bits(HEADER_BITS)
        bps = r.read() + MIN_BITS_PER_VALUE
        remaining -= HEADER_BITS
        r.set_bits(bps)
        target -= min(sorted_count, remaining // bps) * bps
    else:
        r.set_bits(bits_per_unsorted)
    out, acc = [], 0
    while remaining > target:                          # sorted: wrapping u32 sums of the deltas
        acc = (acc + (r.read() & 0xFFFFFFFF)) & 0xFFFFFFFF
        remaining -= r.bits
        out.append(acc)
    r.set_bits(bits_per_unsorted)                      # as PackedLinksIterator::fold does
    while remaining >= r.bits:
        remaining -= r.bits
        out.append(r.read() & 0xFFFFFFFF)
    return out


def packed_links_size(data: bytes, bits_per_unsorted: int, sorted_count: int, total_count: int) -> int:
    """bitpacking_links.rs:112-136: byte size of the first `total_count` links, whatever follows them."""
    if total_count == 0 or not len(data):
        return 0
    ns = min(total_count, sorted_count)
    bits = 0
    if ns:
        bits += HEADER_BITS + ns * ((data[0] & 31) + MIN_BITS_PER_VALUE)
    bits += (total_count - ns) * bits_per_unsorted
    return (bits + 7) // 8


# ------------------------------------------------------------------------------------------------ bitpacking_ordered
class Parameters:
    def __init__(self, length: int, base_bits: int, delta_bits: int, chunk_len_log2: int):
        self.length, self.base_bits, self.delta_bits, self.chunk_len_log2 = int(length), int(base_bits), int(delta_bits), int(chunk_len_log2)

    def chunk_size_bytes(self) -> int:
        return (self.base_bits + self.delta_bits * ((1 << self.chunk_len_log2) - 1) + 7) // 8

    def compressed_size_bytes(self) -> int:
        chunks = -(-self.length // (1 << self.chunk_len_log2))
        return chunks * self.chunk_size_bytes() + TAIL_SIZE

    def valid(self) -> bool:
        return 1 <= self.base_bits <= 64 and 1 <= self.delta_bits <= 56 and self.chunk_len_log2 <= MAX_CHUNK_LEN_LOG2

    def __repr__(self):
        return f"Parameters(length={self.length}, base_bits={self.base_bits}, delta_bits={self.delta_bits}, chunk_len_log2={self.chunk_len_log2})"


def _u64(values) -> np.ndarray:
    return np.asarray(values, dtype=np.uint64).reshape(-1)


def _packed_bits_np(v) -> np.ndarray:
    """packed_bits of each uint64 (binary search on the shifts, exact)"""
    v = np.asarray(v, dtype=np.uint64).copy()
    b = np.zeros(v.shape, np.int64)
    for sh in (32, 16, 8, 4, 2, 1):
        hit = (v >> np.uint64(sh)) != 0
        b += np.where(hit, sh, 0)
        v = np.where(hit, v >> np.uint64(sh), v)
    return b + (v != 0)


def try_all(values) -> list[Parameters]:
    """Parameters::try_all (bitpacking_ordered.rs:212-228)"""
    v = _u64(values)
    last = int(v[-1]) if v.size else 0
    out = []
    for log2 in range(MAX_CHUNK_LEN_LOG2 + 1):
        delta_bits = 1
        if v.size:
            firsts = v[:: 1 << log2]
            lasts = v[np.minimum(np.arange(firsts.size) * (1 << log2) + (1 << log2) - 1, v.size - 1)]
            delta_bits = max(1, int(_packed_bits_np(lasts - firsts).max()))
        p = Parameters(v.size, max(packed_bits(last), 1), delta_bits, log2)
        if 1 <= p.delta_bits <= 56:
            out.append(p)
    return out


def find_best(values) -> Parameters:
    """Parameters::find_best: the first parameter set of minimal size"""
    cands = try_all(values)
    return min(cands, key=lambda p: p.compressed_size_bytes())


def _place_bits(total_bytes: int, pos: np.ndarray, val: np.ndarray, width, words: np.ndarray | None = None) -> np.ndarray:
    """OR `width`-bit values (<= 64 bits) at increasing bit positions into a zeroed little-endian word buffer (LSB first)."""
    if words is None:
        words = np.zeros(total_bytes // 8 + 2, dtype=np.uint64)
    if pos.size:
        pos = pos.astype(np.uint64)
        val = val.astype(np.uint64)
        wi = (pos >> np.uint64(6)).astype(np.int64)
        sh = pos & np.uint64(63)
        lo = val << sh
        spill = (sh > 0) & (sh.astype(np.int64) + np.asarray(width, dtype=np.int64) > 64)
        hi = np.where(spill, val >> np.where(spill, np.uint64(64) - sh, np.uint64(0)), np.uint64(0))
        for idx, part in ((wi, lo), (wi + 1, hi)):
            starts = np.flatnonzero(np.r_[True, idx[1:] != idx[:-1]])
            words[idx[starts]] |= np.bitwise_or.reduceat(part, starts)
    return words


def _bytes_of(words: np.ndarray, total_bytes: int) -> bytearray:
    return bytearray(words.view(np.uint8)[:total_bytes].tobytes())


def compress_with_parameters(values, p: Parameters) -> bytes:
    """bitpacking_ordered.rs:76-104: per chunk the base, the deltas (an incomplete chunk padded with all-ones deltas), byte
    padding; then the 7-byte 0xFF tail."""
    v = _u64(values)
    assert v.size == p.length and p.valid()
    cl = 1 << p.chunk_len_log2
    chunks = -(-v.size // cl)
    if chunks == 0:
        return b"\xff" * TAIL_SIZE
    grid = np.full(chunks * cl, 0, dtype=np.uint64)
    grid[: v.size] = v
    grid = grid.reshape(chunks, cl)
    base = grid[:, 0].copy()
    deltas = grid[:, 1:] - base[:, None]
    flat_pad = np.zeros(chunks * cl, dtype=bool)
    flat_pad[v.size:] = True
    deltas[flat_pad.reshape(chunks, cl)[:, 1:]] = np.uint64(make_bitmask(p.delta_bits))
    assert int(_packed_bits_np(base).max()) <= p.base_bits and (deltas.size == 0 or int(_packed_bits_np(deltas).max()) <= p.delta_bits)
    cbytes = p.chunk_size_bytes()
    start = np.arange(chunks, dtype=np.uint64) * np.uint64(8 * cbytes)
    pos = np.concatenate([start[:, None], start[:, None] + np.uint64(p.base_bits) + np.arange(cl - 1, dtype=np.uint64)[None, :] * np.uint64(p.delta_bits)], axis=1)
    vals = np.concatenate([base[:, None], deltas], axis=1)
    width = np.concatenate([np.full((chunks, 1), p.base_bits), np.full((chunks, cl - 1), p.delta_bits)], axis=1)
    out = _bytes_of(_place_bits(chunks * cbytes, pos.reshape(-1), vals.reshape(-1), width.reshape(-1)), chunks * cbytes)
    out += b"\xff" * TAIL_SIZE
    assert len(out) == p.compressed_size_bytes()
    return bytes(out)


def compress(values, chunk_len_log2: int | None = None) -> tuple[bytes, Parameters]:
    """bitpacking_ordered::compress; chunk_len_log2 forces that chunk length (deltas then as wide as they need)"""
    if chunk_len_log2 is None:
        p = find_best(values)
    else:
        p = [q for q in try_all(values) if q.chunk_len_log2 == chunk_len_log2][0]
    return compress_with_parameters(values, p), p


def _read_le64(data: bytes, off: int) -> int:
    return int.from_bytes(data[off:off + 8], "little")


def read_pair(data: bytes, p: Parameters, index: int):
    """SliceReader::read_pair + Reader::decode_chunk: (value[index], value[index + 1]) or None"""
    if index >= max(p.length - 1, 0):
        return None
    mask = (1 << p.chunk_len_log2) - 1
    cbytes = p.chunk_size_bytes()

    def decode(i):
        c = (i >> p.chunk_len_log2) * cbytes
        base = _read_le64(data, c) & make_bitmask(p.base_bits)
        j = i & mask
        if j == 0:
            return base
        bits = p.base_bits + (j - 1) * p.delta_bits
        return (base + ((_read_le64(data, c + bits // 8) >> (bits % 8)) & make_bitmask(p.delta_bits))) & M64

    return decode(index), decode(index + 1)


# ------------------------------------------------------------------------------------------------ the whole file
def bits_per_unsorted(point_count: int) -> int:
    return max(MIN_BITS_PER_VALUE, packed_bits(max(point_count - 1, 0)))


def _pack_entries(neighbors: np.ndarray, offsets: np.ndarray, sorted_counts: np.ndarray, bpu: int) -> tuple[bytes, np.ndarray]:
    """pack_links over a CSR batch of entries at once: (bytes, byte size of each entry)."""
    cnt = np.diff(offsets).astype(np.int64)
    n_e = cnt.size
    if n_e == 0:
        return b"", np.zeros(0, np.int64)
    ent = np.repeat(np.arange(n_e), cnt)
    k = np.arange(neighbors.size, dtype=np.int64) - np.repeat(offsets[:-1].astype(np.int64), cnt)
    ns = np.minimum(cnt, sorted_counts.astype(np.int64))
    is_sorted = k < ns[ent]
    vals = neighbors.astype(np.uint64)
    # sort the first ns of each entry (one sort of (entry, value) keys), then delta-code them
    sidx = np.flatnonzero(is_sorted)
    se = ent[sidx]
    keyed = np.sort((se.astype(np.uint64) << np.uint64(32)) | vals[sidx])
    sv = keyed & np.uint64(0xFFFFFFFF)
    first = np.r_[True, se[1:] != se[:-1]]
    d = sv.copy()
    d[1:] -= np.where(first[1:], np.uint64(0), sv[:-1])
    deltas = vals.copy()
    deltas[sidx] = d
    maxd = np.zeros(n_e, dtype=np.int64)
    if sidx.size:
        seg = np.flatnonzero(first)
        maxd[se[seg]] = np.maximum.reduceat(_packed_bits_np(d), seg)
    bps = np.maximum(maxd, MIN_BITS_PER_VALUE)
    assert bpu >= int(_packed_bits_np(vals[~is_sorted]).max(initial=0)), "an unsorted link does not fit bits_per_unsorted"
    nbits = np.where(cnt > 0, np.where(ns > 0, HEADER_BITS + ns * bps, 0) + (cnt - ns) * bpu, 0)
    size = (nbits + 7) // 8
    total = int(size.sum())
    start = np.r_[0, np.cumsum(size)[:-1]] * 8
    has_hdr = (cnt > 0) & (ns > 0)
    hdr_e = np.flatnonzero(has_hdr)
    first_bit = start + np.where(has_hdr, HEADER_BITS, 0)
    e_bps = bps[ent]
    e_ns = ns[ent]
    pos_v = first_bit[ent] + np.where(is_sorted, k * e_bps, e_ns * e_bps + (k - e_ns) * bpu)
    words = _place_bits(total, pos_v, deltas, np.where(is_sorted, e_bps, bpu))        # values, then the 5-bit headers
    words = _place_bits(total, start[hdr_e], (bps[hdr_e] - MIN_BITS_PER_VALUE).astype(np.uint64), HEADER_BITS, words)
    return bytes(_bytes_of(words, total)), size


def compress_plain_csr(point_count: int, level_offsets, reindex, neighbors, offsets, m: int, m0: int, chunk_len_log2: int | None = None,
                       batch: int = 1 << 19) -> bytes:
    """GraphLinksFormatParam::Compressed of a graph given in the plain format's arrays (level offsets, reindex, neighbours
    CSR over all (node, level) entries, element offsets) — serializer.rs:62-194 with the same entry order and back_index."""
    n = int(point_count)
    lo = _u64(level_offsets)
    offsets = _u64(offsets)
    neighbors = np.asarray(neighbors, dtype=np.uint32).reshape(-1)
    bpu = bits_per_unsorted(n)
    n_entries = offsets.size - 1
    parts, byte_off = [], [np.zeros(1, np.uint64)]
    total = 0
    for e0 in range(0, n_entries, batch):
        e1 = min(n_entries, e0 + batch)
        sub = offsets[e0:e1 + 1]
        sc = np.where(np.arange(e0, e1) < n, m0, m)
        data, size = _pack_entries(neighbors[int(sub[0]):int(sub[-1])], sub - sub[0], sc, bpu)
        parts.append(data)
        byte_off.append(np.uint64(total) + np.cumsum(size).astype(np.uint64))
        total += len(data)
    boff = np.concatenate(byte_off)
    coff, p = compress(boff, chunk_len_log2)
    hdr = bytearray(64)
    hdr[0:8] = n.to_bytes(8, "little")
    hdr[8:16] = VERSION_COMPRESSED.to_bytes(8, "little")
    hdr[16:24] = int(lo.size).to_bytes(8, "little")
    hdr[24:32] = int(total).to_bytes(8, "little")
    hdr[32:40] = p.length.to_bytes(8, "little")
    hdr[40], hdr[41], hdr[42] = p.base_bits, p.delta_bits, p.chunk_len_log2
    hdr[43:51] = int(m).to_bytes(8, "little")
    hdr[51:59] = int(m0).to_bytes(8, "little")
    return b"".join([bytes(hdr), lo.tobytes(), np.asarray(reindex, dtype=np.uint32).tobytes(), *parts, coff])


def edges_to_plain_arrays(edges):
    """serializer.rs:44-160 for edges[point][level] = links: back_index (points by descending level count; stable, like the
    plain export of the CPU graph), level offsets, reindex, neighbours CSR in entry order, element offsets."""
    n = len(edges)
    nlev = np.array([len(e) for e in edges], dtype=np.int64)
    back = np.argsort(-nlev, kind="stable").astype(np.uint32)
    levels = int(nlev.max()) if n else 0
    by_level = np.bincount(nlev - 1, minlength=levels) if n else np.zeros(0, np.int64)
    lo, tot, suffix = [], 0, n
    for l in range(levels):
        lo.append(tot)
        tot += suffix
        suffix -= int(by_level[l])
    reindex = np.zeros(n, dtype=np.uint32)
    reindex[back] = np.arange(n, dtype=np.uint32)
    nb, off = [], [0]
    for l in range(levels):
        count = int((nlev > l).sum())
        ids = range(count) if l == 0 else back[:count]
        for i in ids:
            links = edges[int(i)][l]
            nb.extend(int(x) for x in links)
            off.append(len(nb))
    return np.array(lo, np.uint64), reindex, np.array(nb, np.uint32), np.array(off, np.uint64)


def serialize_compressed(edges, m: int, m0: int, chunk_len_log2: int | None = None) -> bytes:
    """serialize_graph_links(edges, GraphLinksFormatParam::Compressed, HnswM { m, m0 })"""
    lo, reindex, nb, off = edges_to_plain_arrays(edges)
    return compress_plain_csr(len(edges), lo, reindex, nb, off, m, m0, chunk_len_log2)


def parse_plain(blob):
    """The arrays of a plain links.bin (header.rs:9-20, view.rs:121-135)."""
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    n, levels, n_nb, n_off, pad = (int(x) for x in b[:40].view(np.uint64))
    p = 64
    lo = b[p:p + 8 * levels].view(np.uint64); p += 8 * levels
    reindex = b[p:p + 4 * n].view(np.uint32); p += 4 * n
    nb = b[p:p + 4 * n_nb].view(np.uint32); p += 4 * n_nb + pad
    off = b[p:p + 8 * n_off].view(np.uint64)
    return n, lo, reindex, nb, off


def plain_to_compressed(blob, m: int, m0: int, chunk_len_log2: int | None = None) -> bytes:
    """The compressed file of the graph a plain links.bin holds, with the same back_index (reindex)."""
    n, lo, reindex, nb, off = parse_plain(blob)
    return compress_plain_csr(n, lo, reindex, nb, off, m, m0, chunk_len_log2)


class CompressedLinks:
    """GraphLinksView::load_compressed + links() + point_level(), value by value (view.rs:137-163, 209-263, 354-369)."""

    def __init__(self, blob):
        b = bytes(np.ascontiguousarray(blob, dtype=np.uint8).tobytes()) if not isinstance(blob, (bytes, bytearray)) else bytes(blob)
        u = lambda o: int.from_bytes(b[o:o + 8], "little")
        self.point_count, self.version, self.levels_count, self.total_neighbors_bytes = u(0), u(8), u(16), u(24)
        assert self.version == VERSION_COMPRESSED
        self.params = Parameters(u(32), b[40], b[41], b[42])
        self.m, self.m0 = u(43), u(51)
        assert self.params.valid()
        p = 64
        self.level_offsets = [u(p + 8 * i) for i in range(self.levels_count)] + [self.params.length - 1]
        p += 8 * self.levels_count
        self.reindex = np.frombuffer(b, dtype=np.uint32, count=self.point_count, offset=p)
        p += 4 * self.point_count
        self.neighbors = b[p:p + self.total_neighbors_bytes]
        p += self.total_neighbors_bytes
        self.offsets = b[p:p + self.params.compressed_size_bytes()]
        assert len(self.offsets) == self.params.compressed_size_bytes()
        self.bits_per_unsorted = bits_per_unsorted(self.point_count)

    def level_m(self, level: int) -> int:
        return self.m0 if level == 0 else self.m

    def point_level(self, point: int) -> int:
        r = int(self.reindex[point])
        lo = self.level_offsets
        for level in range(len(lo) - 2):
            if r >= lo[level + 2] - lo[level + 1]:
                return level
        return len(lo) - 2

    def links(self, point: int, level: int) -> list[int]:
        idx = point if level == 0 else self.level_offsets[level] + int(self.reindex[point])
        start, end = read_pair(self.offsets, self.params, idx)
        return iterate_packed_links(self.neighbors[start:end], self.bits_per_unsorted, self.level_m(level))

    def to_edges(self):
        return [[self.links(p, l) for l in range(self.point_level(p) + 1)] for p in range(self.point_count)]


def normalize_links(sorted_count: int, links) -> list[int]:
    """graph_links/mod.rs:97-104"""
    links = [int(x) for x in links]
    links[:sorted_count] = sorted(links[:sorted_count])
    return links


def random_links(rng: np.random.Generator, points_count: int, max_levels_count: int, m: int, m0: int):
    """graph_links/tests.rs:59-80: 1..max_levels_count levels per point, up to 2 x level_m links (payload links), ids repeat."""
    return [[[int(x) for x in rng.integers(0, points_count, int(rng.integers(0, 2 * (m0 if lvl == 0 else m))))]
             for lvl in range(int(rng.integers(1, max_levels_count)))] for _ in range(points_count)]


def serialize_plain(point_count: int, level_offsets, reindex, neighbors, offsets) -> bytes:
    """GraphLinksFormatParam::Plain of the same arrays (header.rs:9-20, serializer.rs:160-175)"""
    lo, nb, off = _u64(level_offsets), np.asarray(neighbors, np.uint32).reshape(-1), _u64(offsets)
    pos = 64 + 8 * lo.size + 4 * int(point_count) + 4 * nb.size
    pad = (8 - pos % 8) % 8
    hdr = np.zeros(8, np.uint64)
    hdr[:5] = [point_count, lo.size, nb.size, off.size, pad]
    return b"".join([hdr.tobytes(), lo.tobytes(), np.asarray(reindex, np.uint32).tobytes(), nb.tobytes(), b"\0" * pad, off.tobytes()])


def synthetic_graph(rng: np.random.Generator, n: int, m: int, m0: int, full: bool = True, max_level: int = 30):
    """A graph of n points with geometric levels (level = floor(-ln(u) / ln(m))) and random links, as the plain format's arrays
    (level offsets, reindex, neighbours, offsets).  full: exactly level_m links per entry; else 0 .. 2 x level_m - 1 (payload
    links), repeats allowed."""
    u = rng.random(n)
    lvl = np.minimum(np.floor(-np.log(np.maximum(u, 1e-300)) / np.log(max(m, 2))), max_level).astype(np.int64)
    levels = int(lvl.max()) + 1 if n else 0
    back = np.argsort(-lvl, kind="stable").astype(np.uint32)
    reindex = np.empty(n, np.uint32)
    reindex[back] = np.arange(n, dtype=np.uint32)
    per_level = np.array([int((lvl >= l).sum()) for l in range(levels)], dtype=np.int64)
    lo = np.r_[0, np.cumsum(per_level)[:-1]].astype(np.uint64)
    lm = np.concatenate([np.full(int(c), m0 if l == 0 else m, np.int64) for l, c in enumerate(per_level)]) if levels else np.zeros(0, np.int64)
    cnt = lm if full else rng.integers(0, 2 * lm)
    off = np.r_[0, np.cumsum(cnt)].astype(np.uint64)
    nb = rng.integers(0, n, int(off[-1]), dtype=np.uint32)
    return lo, reindex, nb, off
