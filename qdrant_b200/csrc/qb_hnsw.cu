// qb_hnsw.cu — device-resident HNSW graph search, batched over queries (BASELINE config 5).
//
// Replaces, for a whole batch of queries at once, the reference's per-query traversal
//   GraphLayers::search            lib/segment/src/index/hnsw_index/graph_layers.rs:530-561
//   search_entry / _on_level       graph_layers.rs:247-316   (greedy descent, beam 1, through the upper levels)
//   search_on_level                graph_layers.rs:108-148   (beam search on level 0)
//   SearchContext::process_candidate / lower_bound           search_context.rs:8-41
//   FilteredScorer::score_points   point_scorer.rs:265-295   (filter, truncate to level_m, score)
// which calls the scorer once per hop with <= m0 ids.  Through a per-call GPU boundary that loop is launch/latency bound
// (round 1: 10x slower than the CPU scorer); here the loop itself runs on the device: one persistent CTA per in-flight
// query (128 threads), graph links resident in HBM, the query in shared memory, the hop's neighbours scored by the CTA's 8-lane groups
// with the SAME bit-exact per-pair arithmetic as the scan kernels (qb_score.cuh), so a hop costs three dependent memory
// round trips (links, visited flags, vectors) and no host interaction.  Throughput comes from many queries in flight
// (SMs x resident CTAs), not from one fast query.
//
// State per query (shared memory): `nearest` = the ef best (score desc, id asc) keys seen so far, kept SORTED, with one
// "expanded" flag each.  In the reference `candidates` (a max-heap) only ever holds points that entered `nearest`; a point
// evicted from `nearest` is strictly worse than lower_bound() and popping it ends the search, so
//   "pop the best candidate; stop if it is below lower_bound"  ==  "take the best not-yet-expanded entry of nearest; stop if none".
// A hop's scored points are merged into the sorted list in parallel (rank = own index + number of keys of the other list
// that are greater), which equals pushing them one by one when scores are distinct; equal scores are ordered by id (the
// reference leaves that to heap order), as everywhere in this library.
// Visited set: one bitmap per resident CTA in HBM/L2 (test-and-set with atomicOr), un-set at the end of a query from a log
// of the ids it touched.
//
// Graph layout: the reference's plain `links.bin` (graph_links/header.rs:9-20, view.rs:121-135, serializer.rs:53-200) is
// taken as is for the upper levels (level_offsets, reindex, neighbors, offsets); level 0 — every hop of the beam search —
// is re-laid at upload as a fixed-stride [n][m0] table so a hop needs ONE coalesced 128-B read instead of offsets -> range.
// The compressed `links.bin` every current index is written in (GraphLinksFormatParam::Compressed, hnsw/build.rs:548-562) is
// decoded on the device into exactly those arrays (qb_hnsw_create_compressed, below), so one traversal serves both formats.
// The kernel (hnsw_search_kernel) and its pieces are in qb_hnsw_traverse.cuh, which the graph build (qb_hnsw_build.cu) shares.
#include <memory>

#include "qb_hnsw_host.cuh"

// ------------------------------------------------------------------------------------------------ host side
// ACORN: to_score holds up to m0 * m0 ids (a passing 1-hop links and at most m0 - a explored lists of m0), its keys sorted in a
// power-of-two buffer; plus to_explore
static uint32_t acorn_hop_cap(uint32_t m0) {
    uint32_t c = HNSW_MAX_LINKS;
    while (c < m0 * m0) c <<= 1;
    return c;
}
static size_t acorn_smem_bytes(uint32_t q_bytes, uint32_t ef, uint32_t hop_cap) {
    return (size_t)((q_bytes + 15u) & ~15u) + (size_t)ef * 16 + (size_t)hop_cap * 16 + 2 * (size_t)((ef + 15u) & ~15u) + HNSW_MAX_LINKS * 4;
}

__global__ void hnsw_links0_kernel(const uint32_t* __restrict__ neighbors, const uint64_t* __restrict__ offsets, uint32_t n, uint32_t m0, uint32_t* __restrict__ links0) {
    const uint64_t total = (uint64_t)n * m0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(i / m0), k = (uint32_t)(i % m0);
        const uint64_t b = offsets[p], e = offsets[p + 1];   // level 0: idx = point id (view.rs:205-206)
        links0[i] = (b + k < e) ? neighbors[b + k] : 0xFFFFFFFFu;
    }
}

// a plain links.bin over `expect` points: the storage's rows, or the points of a multivector collection (`of` names which)
static qb_status hnsw_create_plain_n(qb_storage* s, uint64_t expect, const char* of, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0,
                                     qb_hnsw** out) {
    QB_CHECK(s && links_bin && out, QB_ERR_INVALID, "hnsw_create_plain: null argument");
    *out = nullptr;
    QB_CHECK(m >= 1 && m0 >= 1 && m0 <= HNSW_MAX_LINKS && m <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "hnsw_create_plain: m %u / m0 %u outside [1,%u]", m, m0, HNSW_MAX_LINKS);
    QB_CHECK(n_bytes >= 64, QB_ERR_INVALID, "hnsw_create_plain: %llu bytes is smaller than HeaderPlain", (unsigned long long)n_bytes);
    uint64_t hdr[5];
    memcpy(hdr, links_bin, sizeof(hdr));   // point_count, levels_count, total_neighbors_count, total_offset_count, offsets_padding_bytes
    const uint64_t n = hdr[0], levels = hdr[1], n_nb = hdr[2], n_off = hdr[3], pad = hdr[4];
    QB_CHECK(n == expect, QB_ERR_INVALID, "hnsw_create_plain: graph has %llu points, %s %llu", (unsigned long long)n, of, (unsigned long long)expect);
    QB_CHECK(pad == 0 || pad == 4, QB_ERR_INVALID, "hnsw_create_plain: offsets padding %llu", (unsigned long long)pad);
    QB_CHECK(levels <= 64 && n_off >= n + 1, QB_ERR_INVALID, "hnsw_create_plain: bad header (levels %llu, offsets %llu)", (unsigned long long)levels, (unsigned long long)n_off);
    const uint64_t need = 64 + 8 * levels + 4 * n + 4 * n_nb + pad + 8 * n_off;
    QB_CHECK(n_bytes >= need, QB_ERR_INVALID, "hnsw_create_plain: %llu bytes, header describes %llu", (unsigned long long)n_bytes, (unsigned long long)need);
    const uint8_t* p_lo = links_bin + 64;
    const uint8_t* p_re = p_lo + 8 * levels;
    const uint8_t* p_nb = p_re + 4 * n;
    const uint8_t* p_of = p_nb + 4 * n_nb + pad;
    std::vector<uint64_t> lo(levels + 1);
    {   // level offsets index the offsets table: validate before the device ever follows them
        memcpy(lo.data(), p_lo, 8 * levels);
        for (uint64_t l = 0; l < levels; ++l) QB_CHECK(lo[l] < n_off, QB_ERR_INVALID, "hnsw_create_plain: level offset %llu out of range", (unsigned long long)l);
        lo[levels] = n_off - 1;
    }
    qb_hnsw* g = nullptr;
    QB_TRY(qb_hnsw_new(s, (uint32_t)n, m, m0, std::move(lo), n_off, 0, "hnsw_create_plain", &g));
    g->n_neighbors = n_nb;
    cudaError_t ce = cudaMalloc(&g->d_neighbors, std::max<size_t>(4 * n_nb, 256));
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_plain: cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError())); qb_hnsw_destroy(g); return QB_ERR_OOM; }
    ce = cudaMemcpy(g->d_level_offsets, p_lo, 8 * levels, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, p_re, 4 * n, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_neighbors, p_nb, 4 * n_nb, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_offsets, p_of, 8 * n_off, cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_plain: upload: %s", cudaGetErrorString(ce)); qb_hnsw_destroy(g); return QB_ERR_CUDA; }
    const qb_status st = qb_hnsw_finish_plain(g, "hnsw_create_plain");
    if (st != QB_OK) { qb_hnsw_destroy(g); return st; }
    *out = g;
    return QB_OK;
}

extern "C" qb_status qb_hnsw_create_plain(qb_storage* s, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out) {
    return hnsw_create_plain_n(s, s ? s->count : 0, "storage", links_bin, n_bytes, m, m0, out);
}

qb_status qb_hnsw_new(qb_storage* s, uint32_t n, uint32_t m, uint32_t m0, std::vector<uint64_t> lo, uint64_t n_off, uint64_t tail, const char* who,
                      qb_hnsw** out) {
    *out = nullptr;
    const cudaError_t ce = cudaSetDevice(s->device);
    if (ce != cudaSuccess) { qb_set_error("%s: %s", who, cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    qb_hnsw* g = new qb_hnsw();
    g->st = s; g->n_points = n; g->m = m; g->m0 = m0; g->levels = (uint32_t)(lo.size() - 1);
    g->level_offsets_ext = std::move(lo); g->n_offsets = n_off;
    g->hbm_bytes = 8ull * g->levels + 4ull * n + 8 * (n_off + tail);
    const bool ok = cudaMalloc(&g->d_level_offsets, std::max<size_t>(8ull * g->levels, 256)) == cudaSuccess &&
                    cudaMalloc(&g->d_reindex, std::max<size_t>(4ull * n, 256)) == cudaSuccess &&
                    cudaMalloc(&g->d_offsets, 8 * (n_off + tail) + 256) == cudaSuccess;
    if (!ok) { qb_set_error("%s: cudaMalloc failed: %s", who, cudaGetErrorString(cudaGetLastError())); qb_hnsw_destroy(g); return QB_ERR_OOM; }
    *out = g;
    return QB_OK;
}

qb_status qb_hnsw_finish_plain(qb_hnsw* g, const char* who) {
    const uint64_t n = g->n_points, m0 = g->m0;
    bool ok = cudaMalloc(&g->d_links0, std::max<size_t>((size_t)n * m0 * 4, 256)) == cudaSuccess && cudaMalloc(&g->d_work, 256) == cudaSuccess &&
              cudaMalloc(&g->d_stats, 256) == cudaSuccess;
    if (!ok) { qb_set_error("%s: cudaMalloc failed: %s", who, cudaGetErrorString(cudaGetLastError())); return QB_ERR_OOM; }
    g->hbm_bytes += n * m0 * 4 + 4 * g->n_neighbors;
    cudaError_t ce = cudaMemset(g->d_stats, 0, 256);
    if (ce == cudaSuccess && n) {
        hnsw_links0_kernel<<<hnsw_grid(n * m0, 256, 132 * 16), 256>>>(g->d_neighbors, g->d_offsets, (uint32_t)n, (uint32_t)m0, g->d_links0);
        QB_LAUNCHED();
    }
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce == cudaSuccess) ce = cudaGetLastError();
    if (ce != cudaSuccess) { qb_set_error("%s: upload: %s", who, cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ compressed links.bin
// GraphLinksFormat::Compressed (graph_links/header.rs:22-34, view.rs:137-163, serializer.rs:62-194):
//   HeaderCompressed, 64 B little-endian, nothing after byte 32 aligned:
//     0 point_count | 8 version 0xFFFF_FFFF_FFFF_FF01 | 16 levels_count | 24 total_neighbors_bytes | 32 offsets length (u64) |
//     40 base_bits, 41 delta_bits, 42 chunk_len_log2 (u8 each) | 43 m (u64) | 51 m0 (u64) | 59 five zero bytes
//   then levels_count u64 level offsets, point_count u32 reindex, total_neighbors_bytes of packed links, the compressed offsets.
// Offsets (common/src/bitpacking_ordered.rs:12-39, 165-197, 292-315): chunks of 2^chunk_len_log2 values — a base_bits base,
// then delta_bits deltas from that base, byte-padded — and a 7-byte 0xFF tail.  The values are BYTE offsets into the packed
// links, in the plain format's index space (view.rs:209-218).
// Links of one (node, level) (bitpacking_links.rs:23-133; bit I/O bitpacking.rs:14-186, LSB first): the first
// min(count, level_m) are sorted and delta-coded (wrapping u32 sums) after a 5-bit header `bits_per_sorted - 8`; the rest are
// raw, bits_per_unsorted = max(8, packed_bits(point_count - 1)) bits each (view.rs:155-159).  The count is implicit in the byte
// length L: ns = min(level_m, (8L - 5) / bps), nu = (8L - 5 - ns * bps) / bits_per_unsorted; L == 0: no links.
// Ids may repeat and may be >= point_count (graph_links/tests.rs:59-80); the traversal skips the latter, as for plain graphs.
namespace {

constexpr uint64_t HNSW_VERSION_COMPRESSED = 0xFFFFFFFFFFFFFF01ull;
constexpr uint64_t HNSW_VERSION_COMPRESSED_WITH_VECTORS = 0xFFFFFFFFFFFFFF02ull;
constexpr uint64_t HC_PAD = 16;   // the device copy of the file is padded so the funnel-shift load below never leaves the allocation
enum : uint32_t { HC_OFFSET_PAST_END = 1u, HC_OFFSETS_DECREASE = 2u, HC_REINDEX = 4u };

__device__ __forceinline__ uint64_t hc_min(uint64_t a, uint64_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint64_t hc_mask(uint32_t bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1ull); }

// little-endian u64 at any byte address: two aligned 8-byte loads and a funnel shift
__device__ __forceinline__ uint64_t hc_load_le64(const uint8_t* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t* w = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
    const uint32_t sh = (uint32_t)(a & 7) * 8;
    const uint64_t lo = __ldg(w);
    return sh ? (lo >> sh) | (__ldg(w + 1) << (64 - sh)) : lo;
}

// BitReader::read::<u32> of a `bits`-wide value at bit `bitpos` (bits <= 39, so bitpos % 8 + bits fits one 8-byte word)
__device__ __forceinline__ uint32_t hc_bits(const uint8_t* base, uint64_t bitpos, uint32_t bits) {
    return (uint32_t)((hc_load_le64(base + (bitpos >> 3)) >> (bitpos & 7)) & hc_mask(bits));
}

struct HcOffsets {
    const uint8_t* data;          // compressed offsets
    uint64_t length, chunk_bytes, limit;   // limit = total_neighbors_bytes
    uint32_t base_bits, delta_bits, log2;
};

// Reader::decode_chunk (bitpacking_ordered.rs:292-315), one thread per value; the 7-byte tail keeps every 8-byte read in the data
__global__ void hnsw_c_offsets_kernel(const HcOffsets p, uint64_t* __restrict__ out, uint32_t* __restrict__ flag) {
    const uint64_t base_mask = hc_mask(p.base_bits), delta_mask = hc_mask(p.delta_bits), in_chunk = (1ull << p.log2) - 1ull;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.length; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* c = p.data + (i >> p.log2) * p.chunk_bytes;
        uint64_t v = hc_load_le64(c) & base_mask;
        const uint64_t j = i & in_chunk;
        if (j) {
            const uint64_t bit = p.base_bits + (j - 1) * p.delta_bits;
            v += (hc_load_le64(c + (bit >> 3)) >> (bit & 7)) & delta_mask;
        }
        if (v > p.limit) atomicOr(flag, HC_OFFSET_PAST_END);
        out[i] = v;
    }
}

struct HcLinks {
    const uint8_t* links;         // packed links
    const uint64_t* byte_off;     // decoded offsets [n_entries + 1]
    uint64_t n_entries, limit;
    uint32_t n_points, m, m0, bits_unsorted;
};

// the implicit shape of entry e (iterate_packed_links, bitpacking_links.rs:75-107); entries [0, n_points) are level 0 (view.rs:205-206)
__device__ __forceinline__ void hc_shape(const HcLinks& p, uint64_t e, uint64_t s, uint64_t t, uint32_t& bps, uint64_t& ns, uint64_t& nu) {
    ns = nu = 0; bps = 8;
    if (t == s) return;
    bps = (p.links[s] & 31u) + 8u;
    const uint64_t bits = 8 * (t - s) - 5;
    ns = hc_min(e < p.n_points ? p.m0 : p.m, bits / bps);
    nu = (bits - ns * bps) / p.bits_unsorted;
}

// links per entry (counts[n_entries] = 0, so the exclusive scan ends on the total), and the file's checks that need the device
__global__ void hnsw_c_counts_kernel(const HcLinks p, const uint32_t* __restrict__ reindex, uint64_t* __restrict__ counts, uint32_t* __restrict__ flag) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e <= p.n_entries; e += stride) {
        uint64_t c = 0;
        if (e < p.n_entries) {
            const uint64_t s = p.byte_off[e], t = p.byte_off[e + 1];
            if (t < s) atomicOr(flag, HC_OFFSETS_DECREASE);
            else if (t <= p.limit) { uint32_t bps; uint64_t ns, nu; hc_shape(p, e, s, t, bps, ns, nu); c = ns + nu; }
        }
        counts[e] = c;
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_points; i += stride)
        if (reindex[i] >= p.n_points) atomicOr(flag, HC_REINDEX);
}

// one warp per entry: lane j decodes value j (j + 32, ...) at its own bit position; the sorted part is a warp inclusive scan of
// the deltas (wrapping u32 adds, PackedLinksIterator::next_sorted) with a carry across passes of 32.  bit0: the first sorted value.
__device__ __forceinline__ void hc_decode_warp(const uint8_t* links, uint64_t bit0, uint32_t bps, uint64_t ns, uint64_t nu, uint32_t bits_unsorted,
                                               uint32_t* out, uint32_t lane) {
    uint32_t carry = 0;
    for (uint64_t k0 = 0; k0 < ns; k0 += 32) {
        const uint64_t k = k0 + lane;
        uint32_t v = k < ns ? hc_bits(links, bit0 + k * bps, bps) : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, v, d);
            if (lane >= (uint32_t)d) v += o;
        }
        v += carry;
        if (k < ns) out[k] = v;
        carry = __shfl_sync(0xFFFFFFFFu, v, 31);
    }
    const uint64_t bit1 = bit0 + ns * bps;
    for (uint64_t k = lane; k < nu; k += 32) out[ns + k] = hc_bits(links, bit1 + k * bits_unsorted, bits_unsorted);
}

__global__ void hnsw_c_links_kernel(const HcLinks p, const uint64_t* __restrict__ offsets, uint32_t* __restrict__ neighbors) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t e = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < p.n_entries; e += n_warps) {
        const uint64_t s = p.byte_off[e], t = p.byte_off[e + 1];
        uint32_t bps; uint64_t ns, nu;
        hc_shape(p, e, s, t, bps, ns, nu);
        hc_decode_warp(p.links, 8 * s + 5, bps, ns, nu, p.bits_unsorted, neighbors + offsets[e], lane);
    }
}

// offsets[length .. length + n) = total: an upper-level lookup level_offsets[l] + reindex[p] stays inside the table (and reads an
// empty list) even when a link leads to a point that is not on that level
__global__ void hnsw_c_pad_kernel(uint64_t* offsets, uint64_t length, uint64_t n) {
    const uint64_t total = offsets[length - 1];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) offsets[length + i] = total;
}

// qb_hnsw_links: GraphLinks::links (view.rs:238-263) for a batch of points on one level, from the traversal's own arrays
__global__ void hnsw_links_gather_kernel(const uint32_t* __restrict__ ids, uint32_t n_ids, uint32_t level, uint64_t level_base, uint64_t on_level,
                                         const uint32_t* __restrict__ reindex, const uint64_t* __restrict__ offsets, uint64_t n_offsets,
                                         const uint32_t* __restrict__ neighbors, uint64_t n_neighbors, uint32_t cap, uint32_t* __restrict__ out,
                                         uint32_t* __restrict__ counts, uint32_t* __restrict__ flag) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_ids; i += gridDim.x * blockDim.x) {
        const uint32_t id = ids[i];
        counts[i] = 0;
        uint64_t idx = id;
        if (level) {
            const uint32_t r = reindex[id];
            if (r >= on_level) { atomicOr(flag, 1u); continue; }   // point_level(id) < level (view.rs:354-369)
            idx = level_base + r;
        }
        if (idx + 1 >= n_offsets) { atomicOr(flag, 2u); continue; }
        const uint64_t b = offsets[idx], e = offsets[idx + 1];
        if (b > e || e > n_neighbors) { atomicOr(flag, 2u); continue; }
        counts[i] = (uint32_t)hc_min(e - b, 0xFFFFFFFFull);
        const uint64_t n = hc_min(e - b, cap);
        for (uint64_t k = 0; k < n; ++k) out[(size_t)i * cap + k] = neighbors[b + k];
    }
}

// the fields HeaderCompressed and HeaderCompressedWithVectors share (bytes 0-58), then what hc_check derives from them
struct HcHeader {
    uint64_t n, version, levels, nb_bytes, length, m, m0;
    uint32_t base_bits, delta_bits, log2;
    uint64_t body, chunk_bytes, used;   // where the links / records start, one chunk of offsets, the bytes the file's parts take
    uint32_t bits_unsorted;
    std::vector<uint64_t> lo;           // the level offsets with the extra last element (read_level_offsets, view.rs:381-393)
};

HcHeader hc_header(const uint8_t* bytes) {
    auto u64_at = [&](uint64_t o) { uint64_t v; memcpy(&v, bytes + o, 8); return v; };   // the file is little-endian, like every host this builds for
    HcHeader h{};
    h.n = u64_at(0); h.version = u64_at(8); h.levels = u64_at(16); h.nb_bytes = u64_at(24); h.length = u64_at(32); h.m = u64_at(43); h.m0 = u64_at(51);
    h.base_bits = bytes[40]; h.delta_bits = bytes[41]; h.log2 = bytes[42];
    return h;
}

// the checks both compressed formats make after their own: the counts, the offsets parameters, the parts' sizes against n_bytes, the level
// offsets.  head: the header's size; align: the links / records start at a file offset that is a multiple of it; after: what precedes
// the offsets ("links" / "records"), for the messages
qb_status hc_check(HcHeader& h, const uint8_t* bytes, uint64_t n_bytes, uint64_t head, uint64_t align, uint64_t expect, const char* of, const char* who,
                   const char* after) {
    const uint64_t n = h.n, levels = h.levels, nb_bytes = h.nb_bytes, length = h.length, m = h.m, m0 = h.m0;
    const uint32_t base_bits = h.base_bits, delta_bits = h.delta_bits, log2 = h.log2;
    QB_CHECK(n == expect, QB_ERR_INVALID, "%s: graph has %llu points, %s %llu", who, (unsigned long long)n, of, (unsigned long long)expect);
    QB_CHECK(n <= 0xFFFFFFFFull, QB_ERR_INVALID, "%s: %llu points", who, (unsigned long long)n);
    QB_CHECK(m >= 1 && m0 >= 1, QB_ERR_INVALID, "%s: m %llu / m0 %llu", who, (unsigned long long)m, (unsigned long long)m0);
    QB_CHECK(m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "%s: m %llu / m0 %llu outside [1,%u]", who, (unsigned long long)m,
             (unsigned long long)m0, HNSW_MAX_LINKS);
    QB_CHECK(levels <= 64 && (levels >= 1 || n == 0), QB_ERR_INVALID, "%s: %llu levels", who, (unsigned long long)levels);
    // Parameters::validate (bitpacking_ordered.rs:165-180)
    QB_CHECK(base_bits >= 1 && base_bits <= 64 && delta_bits >= 1 && delta_bits <= 56 && log2 <= 7, QB_ERR_INVALID,
             "%s: offsets parameters base_bits %u delta_bits %u chunk_len_log2 %u", who, base_bits, delta_bits, log2);
    const uint64_t body = h.body = round_up_u64(head + 8 * levels + 4 * n, align);
    QB_CHECK(body <= n_bytes && nb_bytes <= n_bytes - body, QB_ERR_INVALID, "%s: %llu bytes, header describes %llu before the offsets", who,
             (unsigned long long)n_bytes, (unsigned long long)(body + nb_bytes));
    const uint64_t rest = n_bytes - body - nb_bytes;
    const uint64_t chunk_bytes = h.chunk_bytes = ceil_div_u64(base_bits + (uint64_t)delta_bits * ((1ull << log2) - 1), 8);
    const uint64_t chunks = length / (1ull << log2) + ((length & ((1ull << log2) - 1)) ? 1 : 0);
    QB_CHECK(length >= 1 && chunks <= rest / chunk_bytes && chunks * chunk_bytes + 7 <= rest, QB_ERR_INVALID,
             "%s: %llu offsets do not fit the %llu bytes after the %s", who, (unsigned long long)length, (unsigned long long)rest, after);
    h.used = body + nb_bytes + chunks * chunk_bytes + 7;
    // level 0 is the first n entries, every level's range inside the table
    std::vector<uint64_t>& lo = h.lo;
    lo.resize(levels + 1);
    memcpy(lo.data(), bytes + head, 8 * levels);
    lo[levels] = length - 1;
    for (uint64_t l = 0; l < levels; ++l)
        QB_CHECK(lo[l] <= lo[l + 1] && (l != 0 || (lo[0] == 0 && lo[1] == n)), QB_ERR_INVALID, "%s: level offset %llu (%llu) out of range", who,
                 (unsigned long long)l, (unsigned long long)lo[l]);
    h.bits_unsorted = std::max<uint32_t>(8, n > 1 ? 64 - __builtin_clzll(n - 1) : 0);
    return QB_OK;
}

}  // namespace

// a compressed links.bin over `expect` points, as hnsw_create_plain_n
static qb_status hnsw_create_compressed_n(qb_storage* s, uint64_t expect, const char* of, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out) {
    const char* who = "hnsw_create_compressed";
    QB_CHECK(s && bytes && out, QB_ERR_INVALID, "hnsw_create_compressed: null argument");
    *out = nullptr;
    QB_CHECK(n_bytes >= 64, QB_ERR_INVALID, "hnsw_create_compressed: %llu bytes is smaller than HeaderCompressed", (unsigned long long)n_bytes);
    HcHeader h = hc_header(bytes);
    QB_CHECK(h.version != HNSW_VERSION_COMPRESSED_WITH_VECTORS, QB_ERR_UNSUPPORTED,
             "hnsw_create_compressed: CompressedWithVectors (inline storage) graphs are searched from the quantized vectors stored with the links "
             "(graph_layers.rs:336-388), a different algorithm; this loader takes GraphLinksFormat::Compressed");
    QB_CHECK(h.version == HNSW_VERSION_COMPRESSED, QB_ERR_INVALID, "hnsw_create_compressed: version word %016llx is not HEADER_VERSION_COMPRESSED (a plain links.bin?)",
             (unsigned long long)h.version);
    QB_TRY(hc_check(h, bytes, n_bytes, 64, 1, expect, of, who, "links"));
    const uint64_t n = h.n, levels = h.levels, length = h.length;

    qb_hnsw* g = nullptr;
    QB_TRY(qb_hnsw_new(s, (uint32_t)n, (uint32_t)h.m, (uint32_t)h.m0, std::move(h.lo), length, n, who, &g));
    std::unique_ptr<qb_hnsw, decltype(&qb_hnsw_destroy)> guard(g, qb_hnsw_destroy);
    auto fail = [&](qb_status st, const char* what, cudaError_t e) {
        qb_set_error("hnsw_create_compressed: %s: %s", what, cudaGetErrorString(e));
        return st;
    };
    HnswScratch tmp;
    uint8_t* d_file = nullptr; uint64_t* d_byte_off = nullptr; uint64_t* d_counts = nullptr; uint32_t* d_flag = nullptr;
    bool ok = tmp.alloc((void**)&d_file, h.used + HC_PAD) == cudaSuccess && tmp.alloc((void**)&d_byte_off, 8 * length) == cudaSuccess &&
              tmp.alloc((void**)&d_counts, 8 * length) == cudaSuccess && tmp.alloc((void**)&d_flag, 4) == cudaSuccess;
    if (!ok) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    // the file goes to HBM once; everything below reads it there
    cudaError_t ce = cudaMemcpy(d_file, bytes, h.used, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(d_file + h.used, 0, HC_PAD);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_level_offsets, d_file + 64, 8 * levels, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, d_file + 64 + 8 * levels, 4 * n, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(d_flag, 0, 4);
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "upload", ce);

    HcOffsets po{d_file + h.body + h.nb_bytes, length, h.chunk_bytes, h.nb_bytes, h.base_bits, h.delta_bits, h.log2};
    hnsw_c_offsets_kernel<<<hnsw_grid(length, 256, 132 * 16), 256>>>(po, d_byte_off, d_flag);
    QB_LAUNCHED();
    HcLinks pl{d_file + h.body, d_byte_off, length - 1, h.nb_bytes, (uint32_t)n, (uint32_t)h.m, (uint32_t)h.m0, h.bits_unsorted};
    hnsw_c_counts_kernel<<<hnsw_grid(std::max<uint64_t>(length, n), 256, 132 * 16), 256>>>(pl, g->d_reindex, d_counts, d_flag);
    QB_LAUNCHED();
    uint32_t flag = 0;
    QB_TRY(hnsw_link_offsets(g, d_counts, length, tmp, who, "decode", d_flag, &flag, [&](const uint64_t* d_offsets, uint32_t* d_neighbors) {
        hnsw_c_links_kernel<<<hnsw_grid(length - 1, 8, 132 * 32), 256>>>(pl, d_offsets, d_neighbors);
        QB_LAUNCHED();
    }));
    QB_CHECK(!flag, QB_ERR_INVALID, "hnsw_create_compressed: %s", (flag & HC_OFFSET_PAST_END) ? "a links offset lies past total_neighbors_bytes"
                                                                : (flag & HC_OFFSETS_DECREASE) ? "links offsets decrease"
                                                                                               : "a reindex entry is >= point_count");
    hnsw_c_pad_kernel<<<hnsw_grid(n, 256, 132 * 4), 256>>>(g->d_offsets, length, n);
    QB_LAUNCHED();
    QB_TRY(qb_hnsw_finish_plain(g, who));
    *out = guard.release();
    return QB_OK;
}

extern "C" qb_status qb_hnsw_create_compressed(qb_storage* s, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out) {
    return hnsw_create_compressed_n(s, s ? s->count : 0, "storage", bytes, n_bytes, out);
}

// ------------------------------------------------------------------------------------------------ graphs over multivector points
// The graph of a multivector named vector links POINTS; the scorer behind its search is MaxSim over each point's token rows
// (MultiMetricQueryScorer, multi_metric_query_scorer.rs; QuantizedMultivectorStorage, quantized_multivector_storage/mod.rs:328-352).
// The loaders are the regular ones with the point count taken from the collection, plus the token offsets on the device.
qb_status qb_hnsw_mv_check(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const char* who) {
    QB_CHECK(s && point_offsets, QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK((s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32) || s->kind == QB_KIND_SQ8, QB_ERR_UNSUPPORTED,
             "%s: device MaxSim traversal supports dense f32 and SQ8 token storages", who);
    // the checks qb_search_maxsim makes (maxsim_run)
    for (uint32_t p = 0; p < n_points; ++p) QB_CHECK(point_offsets[p] <= point_offsets[p + 1], QB_ERR_INVALID, "%s: point_offsets not ascending at %u", who, p);
    QB_CHECK(point_offsets[n_points] <= s->count, QB_ERR_INVALID, "%s: point_offsets end %u beyond the %llu stored vectors", who, point_offsets[n_points],
             (unsigned long long)s->count);
    return QB_OK;
}

qb_status qb_hnsw_mv_upload(const uint32_t* point_offsets, uint32_t n_points, const char* who, uint32_t** d_tok) {
    const size_t bytes = 4ull * ((size_t)n_points + 1);
    *d_tok = nullptr;
    cudaError_t ce = cudaMalloc(d_tok, bytes);
    if (ce == cudaSuccess) ce = cudaMemcpy(*d_tok, point_offsets, bytes, cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) {
        qb_set_error("%s: offsets upload: %s", who, cudaGetErrorString(ce));
        cudaFree(*d_tok);
        *d_tok = nullptr;
        return ce == cudaErrorMemoryAllocation ? QB_ERR_OOM : QB_ERR_CUDA;
    }
    return QB_OK;
}

void qb_hnsw_mv_attach(qb_hnsw* g, uint32_t* d_tok, uint32_t n_points) {
    g->d_mv_tok = d_tok;
    g->hbm_bytes += 4ull * ((size_t)n_points + 1);
}

// a loader's graph (create) over the points of a multivector collection, with their token offsets attached
template <class Create>
static qb_status hnsw_create_mv(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const char* who, qb_hnsw** out, Create create) {
    QB_CHECK(out, QB_ERR_INVALID, "%s: null argument", who);
    *out = nullptr;
    QB_TRY(qb_hnsw_mv_check(tokens, point_offsets, n_points, who));
    qb_hnsw* g = nullptr;
    QB_TRY(create(&g));
    uint32_t* d_tok = nullptr;
    const qb_status st = qb_hnsw_mv_upload(point_offsets, n_points, who, &d_tok);
    if (st != QB_OK) { qb_hnsw_destroy(g); return st; }
    qb_hnsw_mv_attach(g, d_tok, n_points);
    *out = g;
    return QB_OK;
}

extern "C" qb_status qb_hnsw_create_plain_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const uint8_t* links_bin,
                                                      uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out) {
    return hnsw_create_mv(tokens, point_offsets, n_points, "hnsw_create_plain_multivector", out,
                          [&](qb_hnsw** g) { return hnsw_create_plain_n(tokens, n_points, "collection", links_bin, n_bytes, m, m0, g); });
}

extern "C" qb_status qb_hnsw_create_compressed_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const uint8_t* bytes,
                                                           uint64_t n_bytes, qb_hnsw** out) {
    return hnsw_create_mv(tokens, point_offsets, n_points, "hnsw_create_compressed_multivector", out,
                          [&](qb_hnsw** g) { return hnsw_create_compressed_n(tokens, n_points, "collection", bytes, n_bytes, g); });
}

// ------------------------------------------------------------------------------------------------ compressed links.bin with vectors
// GraphLinksFormat::CompressedWithVectors (header.rs:37-70, serializer.rs:32-49,91-171, view.rs:165-207,276-352), written for indexes
// with inline storage:
//   HeaderCompressedWithVectors, 80 B: bytes 0-58 as HeaderCompressed (version 0xFFFF_FFFF_FFFF_FF02), then base_vector_layout
//   {u64 size, u8 align} at 59, link_vector_layout at 68, 3 zero bytes; level offsets, reindex, zero padding up to a FILE offset that
//   is a multiple of max(base align, link align), total_neighbors_bytes of records, the compressed byte offsets.
//   A record: [base vector, level 0 only][varint link count][packed links][pad to link align][count x link vector][level 0: pad to
//   base align]; the alignments are relative to the start of the records.  The count is explicit (packed_links_size uses it).
// The links are decoded once into the plain arrays the regular traversal reads (so qb_hnsw_links / _export_plain / the HNSW, ACORN
// and custom searches work on this handle unchanged); the records stay resident for qb_hnsw_search_with_vectors_batch, with each
// entry's link-vector offset and each point's base-vector offset.
namespace {

enum : uint32_t { HV_RECORD = 8u, HV_TOO_WIDE = 16u };

struct HvShape {
    const uint8_t* links;         // the records
    const uint64_t* byte_off;     // decoded offsets [n_entries + 1]
    uint64_t n_entries, limit, base_size, link_size;
    uint32_t n_points, m, m0, bits_unsorted, link_align;
};

// per entry: link count, where its packed links and link vectors start; every part checked to lie inside the record
__global__ void hnsw_v_shape_kernel(const HvShape p, const uint32_t* __restrict__ reindex, uint64_t* __restrict__ counts, uint64_t* __restrict__ lstart,
                                    uint64_t* __restrict__ lvoff, uint32_t* __restrict__ flag) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e <= p.n_entries; e += stride) {
        uint64_t c = 0, ls = 0, lv = 0;
        if (e < p.n_entries) {
            const uint64_t s = p.byte_off[e], t = p.byte_off[e + 1];
            if (t < s) atomicOr(flag, HC_OFFSETS_DECREASE);
            else if (t <= p.limit) {
                uint64_t pos = s + (e < p.n_points ? p.base_size : 0);
                bool ok = pos <= t, done = false;
                uint64_t cnt = 0;
                for (uint32_t i = 0; ok && !done && i < 10; ++i) {   // u64::decode_var
                    if (pos >= t) { ok = false; break; }
                    const uint32_t b = p.links[pos++];
                    cnt |= (uint64_t)(b & 127u) << (7 * i);
                    done = (b & 128u) == 0;
                }
                ok = ok && done;
                const bool wide = ok && cnt > HNSW_MAX_LIST;
                if (wide) ok = false;
                else if (ok && cnt) {
                    if (pos >= t) ok = false;
                    else {   // packed_links_size (bitpacking_links.rs:112-136)
                        const uint64_t bps = (p.links[pos] & 31u) + 8u, ns = hc_min(cnt, e < p.n_points ? p.m0 : p.m);
                        ls = pos;
                        pos += (5 + ns * bps + (cnt - ns) * p.bits_unsorted + 7) / 8;
                    }
                }
                if (ok) {
                    pos = (pos + p.link_align - 1) / p.link_align * p.link_align;
                    ok = pos <= t && cnt * p.link_size <= t - pos;
                }
                if (ok) { c = cnt; lv = pos; }
                else atomicOr(flag, wide ? HV_TOO_WIDE : HV_RECORD);
            }
        }
        counts[e] = c;
        if (e < p.n_entries) { lstart[e] = ls; lvoff[e] = lv; }
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_points; i += stride)
        if (reindex[i] >= p.n_points) atomicOr(flag, HC_REINDEX);
}

__global__ void hnsw_v_links_kernel(const HvShape p, const uint64_t* __restrict__ lstart, const uint64_t* __restrict__ offsets, uint32_t* __restrict__ neighbors) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t e = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < p.n_entries; e += n_warps) {
        const uint64_t cnt = offsets[e + 1] - offsets[e];
        if (!cnt) continue;
        const uint64_t ls = lstart[e];
        const uint64_t ns = hc_min(cnt, e < p.n_points ? p.m0 : p.m);
        hc_decode_warp(p.links, 8 * ls + 5, (p.links[ls] & 31u) + 8u, ns, cnt - ns, p.bits_unsorted, neighbors + offsets[e], lane);
    }
}

}  // namespace

extern "C" qb_status qb_hnsw_create_with_vectors(qb_storage* s, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out) {
    QB_CHECK(s && bytes && out, QB_ERR_INVALID, "hnsw_create_with_vectors: null argument");
    *out = nullptr;
    QB_CHECK(n_bytes >= 80, QB_ERR_INVALID, "hnsw_create_with_vectors: %llu bytes is smaller than HeaderCompressedWithVectors", (unsigned long long)n_bytes);
    const char* who = "hnsw_create_with_vectors";
    HcHeader h = hc_header(bytes);
    uint64_t base_size, link_size;
    memcpy(&base_size, bytes + 59, 8); memcpy(&link_size, bytes + 68, 8);
    const uint32_t base_align = bytes[67], link_align = bytes[76];
    QB_CHECK(h.version == HNSW_VERSION_COMPRESSED_WITH_VECTORS, QB_ERR_INVALID,
             "hnsw_create_with_vectors: version word %016llx is not HEADER_VERSION_COMPRESSED_WITH_VECTORS (a Compressed or plain links.bin?)",
             (unsigned long long)h.version);
    QB_CHECK(s->kind == QB_KIND_SQ8, QB_ERR_UNSUPPORTED,
             "hnsw_create_with_vectors: the link vectors are read as rows of the bound storage, which must be scalar-quantized (SQ8)");
    // Layout::from_size_align (header.rs:63-69): a power-of-two alignment
    QB_CHECK(base_align && !(base_align & (base_align - 1)) && link_align && !(link_align & (link_align - 1)), QB_ERR_INVALID,
             "hnsw_create_with_vectors: vector alignments %u / %u are not powers of two", base_align, link_align);
    QB_CHECK(base_size != 2ull * s->dim && base_size != s->dim, QB_ERR_UNSUPPORTED,
             "hnsw_create_with_vectors: base vectors of %llu bytes at dim %u are f16 or u8; only f32 base vectors are supported",
             (unsigned long long)base_size, s->dim);
    QB_CHECK(base_size == 4ull * s->dim, QB_ERR_INVALID, "hnsw_create_with_vectors: base vectors of %llu bytes, dim %u", (unsigned long long)base_size, s->dim);
    QB_CHECK(link_size == 4ull + s->actual_dim, QB_ERR_INVALID, "hnsw_create_with_vectors: link vectors of %llu bytes, the storage's rows have %u",
             (unsigned long long)link_size, 4u + s->actual_dim);
    QB_TRY(hc_check(h, bytes, n_bytes, 80, std::max(base_align, link_align), s->count, "storage", who, "records"));
    const uint64_t n = h.n, levels = h.levels, nb_bytes = h.nb_bytes, length = h.length;

    qb_hnsw* g = nullptr;
    QB_TRY(qb_hnsw_new(s, (uint32_t)n, (uint32_t)h.m, (uint32_t)h.m0, std::move(h.lo), length, n, who, &g));
    std::unique_ptr<qb_hnsw, decltype(&qb_hnsw_destroy)> guard(g, qb_hnsw_destroy);
    g->link_size = (uint32_t)link_size;
    auto fail = [&](qb_status st, const char* what, cudaError_t e) {
        qb_set_error("hnsw_create_with_vectors: %s: %s", what, cudaGetErrorString(e));
        return st;
    };
    HnswScratch tmp;
    uint8_t* d_file = nullptr; uint64_t *d_byte_off = nullptr, *d_counts = nullptr, *d_lstart = nullptr; uint32_t* d_flag = nullptr;
    bool ok = cudaMalloc(&g->d_blob, nb_bytes + HC_PAD) == cudaSuccess && cudaMalloc(&g->d_lvoff, 8 * (length + n) + 256) == cudaSuccess &&
              cudaMalloc(&g->d_boff, std::max<size_t>(8 * n, 256)) == cudaSuccess &&
              tmp.alloc((void**)&d_file, h.used + HC_PAD) == cudaSuccess && tmp.alloc((void**)&d_byte_off, 8 * length) == cudaSuccess &&
              tmp.alloc((void**)&d_counts, 8 * length) == cudaSuccess && tmp.alloc((void**)&d_lstart, 8 * length) == cudaSuccess &&
              tmp.alloc((void**)&d_flag, 4) == cudaSuccess;
    if (!ok) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    g->hbm_bytes += (nb_bytes + HC_PAD) + 8 * (length + n) + 8 * n;
    cudaError_t ce = cudaMemcpy(d_file, bytes, h.used, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(d_file + h.used, 0, HC_PAD);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_level_offsets, d_file + 80, 8 * levels, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, d_file + 80 + 8 * levels, 4 * n, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_blob, d_file + h.body, nb_bytes, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(g->d_blob + nb_bytes, 0, HC_PAD);
    if (ce == cudaSuccess) ce = cudaMemset(g->d_lvoff, 0, 8 * (length + n) + 256);
    if (ce == cudaSuccess) ce = cudaMemset(d_flag, 0, 4);
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "upload", ce);

    HcOffsets po{d_file + h.body + nb_bytes, length, h.chunk_bytes, nb_bytes, h.base_bits, h.delta_bits, h.log2};
    hnsw_c_offsets_kernel<<<hnsw_grid(length, 256, 132 * 16), 256>>>(po, d_byte_off, d_flag);
    QB_LAUNCHED();
    HvShape pv{d_file + h.body, d_byte_off, length - 1, nb_bytes, base_size, link_size, (uint32_t)n, (uint32_t)h.m, (uint32_t)h.m0, h.bits_unsorted, link_align};
    hnsw_v_shape_kernel<<<hnsw_grid(std::max<uint64_t>(length, n), 256, 132 * 16), 256>>>(pv, g->d_reindex, d_counts, d_lstart, g->d_lvoff, d_flag);
    QB_LAUNCHED();
    uint32_t flag = 0;
    QB_TRY(hnsw_link_offsets(g, d_counts, length, tmp, who, "decode", d_flag, &flag, [&](const uint64_t* d_offsets, uint32_t* d_neighbors) {
        hnsw_v_links_kernel<<<hnsw_grid(length - 1, 8, 132 * 32), 256>>>(pv, d_lstart, d_offsets, d_neighbors);
        QB_LAUNCHED();
    }));
    if (flag) {
        qb_set_error("hnsw_create_with_vectors: %s", (flag & HC_OFFSET_PAST_END) ? "a record offset lies past total_neighbors_bytes"
                                                    : (flag & HC_OFFSETS_DECREASE) ? "record offsets decrease"
                                                    : (flag & HC_REINDEX)          ? "a reindex entry is >= point_count"
                                                    : (flag & HV_RECORD)           ? "a record's count, links or link vectors run past its end"
                                                                                   : "a list has more than 128 links");
        return flag == HV_TOO_WIDE ? QB_ERR_UNSUPPORTED : QB_ERR_INVALID;
    }
    if (n && (ce = cudaMemcpy(g->d_boff, d_byte_off, 8 * n, cudaMemcpyDeviceToDevice)) != cudaSuccess) return fail(QB_ERR_CUDA, "decode", ce);
    hnsw_c_pad_kernel<<<hnsw_grid(n, 256, 132 * 4), 256>>>(g->d_offsets, length, n);
    QB_LAUNCHED();
    QB_TRY(qb_hnsw_finish_plain(g, who));
    *out = guard.release();
    return QB_OK;
}

extern "C" qb_status qb_hnsw_links(const qb_hnsw* g, uint32_t level, const uint32_t* ids, uint32_t n_ids, uint32_t cap, uint32_t* out, uint32_t* counts) {
    QB_CHECK(g && (ids || n_ids == 0) && (counts || n_ids == 0) && (out || cap == 0 || n_ids == 0), QB_ERR_INVALID, "hnsw_links: null argument");
    QB_CHECK(level < g->levels, QB_ERR_INVALID, "hnsw_links: level %u but the graph has %u levels", level, g->levels);
    for (uint32_t i = 0; i < n_ids; ++i) QB_CHECK(ids[i] < g->n_points, QB_ERR_INVALID, "hnsw_links: point %u out of range", ids[i]);
    if (n_ids == 0) return QB_OK;
    // a point is on `level` iff its reindex is below every level's point count up to there (point_level, view.rs:354-369)
    const std::vector<uint64_t>& lo = g->level_offsets_ext;
    uint64_t on_level = ~0ull;
    for (uint32_t l = 1; l <= level; ++l) on_level = std::min<uint64_t>(on_level, lo[l + 1] >= lo[l] ? lo[l + 1] - lo[l] : 0);
    QB_CUDA(cudaSetDevice(g->st->device));
    HnswScratch tmp;
    uint32_t *d_ids = nullptr, *d_out = nullptr, *d_counts = nullptr, *d_flag = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_ids, 4ull * n_ids));
    QB_CUDA(tmp.alloc((void**)&d_out, 4ull * n_ids * cap));
    QB_CUDA(tmp.alloc((void**)&d_counts, 4ull * n_ids));
    QB_CUDA(tmp.alloc((void**)&d_flag, 4));
    QB_CUDA(cudaMemcpy(d_ids, ids, 4ull * n_ids, cudaMemcpyHostToDevice));
    QB_CUDA(cudaMemset(d_flag, 0, 4));
    hnsw_links_gather_kernel<<<hnsw_grid(n_ids, 128, 132 * 8), 128>>>(d_ids, n_ids, level, level ? lo[level] : 0, on_level, g->d_reindex, g->d_offsets, g->n_offsets,
                                                                    g->d_neighbors, g->n_neighbors, cap, d_out, d_counts, d_flag);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    uint32_t flag = 0;
    QB_CUDA(cudaMemcpy(&flag, d_flag, 4, cudaMemcpyDeviceToHost));
    QB_CHECK(!(flag & 1u), QB_ERR_INVALID, "hnsw_links: a point's top level is below %u", level);
    QB_CHECK(!(flag & 2u), QB_ERR_INVALID, "hnsw_links: the graph's offsets point outside its tables");
    QB_CUDA(cudaMemcpy(counts, d_counts, 4ull * n_ids, cudaMemcpyDeviceToHost));
    if (cap) QB_CUDA(cudaMemcpy(out, d_out, 4ull * n_ids * cap, cudaMemcpyDeviceToHost));
    return QB_OK;
}

extern "C" void qb_hnsw_destroy(qb_hnsw* g) {
    if (!g) return;
    if (g->st) cudaSetDevice(g->st->device);
    cudaDeviceSynchronize();
    cudaFree(g->d_links0); cudaFree(g->d_level_offsets); cudaFree(g->d_reindex); cudaFree(g->d_neighbors); cudaFree(g->d_offsets);
    cudaFree(g->d_visited); cudaFree(g->d_vlog); cudaFree(g->d_work); cudaFree(g->d_stats);
    cudaFree(g->d_blob); cudaFree(g->d_lvoff); cudaFree(g->d_boff); cudaFree(g->d_mv_tok);
    cudaGetLastError();
    delete g;
}

extern "C" qb_status qb_hnsw_info(const qb_hnsw* g, uint32_t* n_points, uint32_t* levels, uint64_t* hbm_bytes) {
    QB_CHECK(g, QB_ERR_INVALID, "hnsw_info: null graph");
    if (n_points) *n_points = g->n_points;
    if (levels) *levels = g->levels;
    if (hbm_bytes) *hbm_bytes = g->hbm_bytes;
    return QB_OK;
}

// queries already encoded (d_q_enc / d_q_off); results to device buffers; enqueued on `stream`, no synchronisation
qb_status qb_hnsw_launch(qb_hnsw* g, const void* d_q_enc, const float* d_q_off, uint32_t nq, uint32_t top, uint32_t ef, uint32_t entry, uint32_t entry_level,
                         const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts, cudaStream_t stream, int algo, const QbHnswCustom* custom,
                         const QbHnswMaxsim* maxsim) {
    qb_storage* s = g->st;
    QB_CHECK(!maxsim == !g->d_mv_tok, QB_ERR_UNSUPPORTED,
             maxsim ? "hnsw_search_maxsim: the graph is not over multivector points (load it with qb_hnsw_create_*_multivector)"
                    : "hnsw_search: the graph is over multivector points; search it with qb_hnsw_search_maxsim_batch / _maxsim_custom_batch");
    const bool mv_custom = custom && maxsim;
    QB_CHECK(algo == ALGO_HNSW || algo == ALGO_ACORN, QB_ERR_INVALID, "hnsw_search: algorithm %d is neither QB_HNSW_ALGO_HNSW nor QB_HNSW_ALGO_ACORN", algo);
    QB_CHECK(entry < g->n_points, QB_ERR_INVALID, "hnsw_search: entry point %u out of range", entry);
    QB_CHECK(entry_level < std::max<uint32_t>(g->levels, 1), QB_ERR_INVALID, "hnsw_search: entry level %u but the graph has %u levels", entry_level, g->levels);
    ef = std::max(ef, top);   // graph_layers.rs:551
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "hnsw_search: ef %u > %u", ef, HNSW_MAX_EF);
    int kind;
    if (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32) kind = s->dim >= 32 ? HK_DENSE_AVX : HK_DENSE_SMALL;
    else if (s->kind == QB_KIND_SQ8) kind = ((uint64_t)s->actual_dim * 127ull * 127ull >= (1ull << 24)) ? HK_SQ8_LANEX : HK_SQ8;
    else if (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_U8 && !maxsim) kind = s->dim >= 32 ? HK_U8 : HK_U8_SMALL;
    else {
        qb_set_error("hnsw_search: device traversal supports dense f32, Uint8 and SQ8 storages, MaxSim dense f32 and SQ8 tokens (others go through "
                     "qb_score_points per hop)");
        return QB_ERR_UNSUPPORTED;
    }
    const int metric = hnsw_metric(s);
    HnswParams p{};
    p.links0 = g->d_links0; p.level_offsets = g->d_level_offsets; p.reindex = g->d_reindex; p.neighbors = g->d_neighbors; p.offsets = g->d_offsets;
    p.n_points = g->n_points; p.m = g->m; p.m0 = g->m0; p.levels = g->levels;
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim;
    p.codes = s->d_codes; p.voff = s->d_voff; p.ad = s->actual_dim; p.multiplier = s->multiplier; p.l1 = (s->qdist == QB_QD_L1) ? 1 : 0;
    p.q_enc = reinterpret_cast<const uint8_t*>(d_q_enc); p.q_bytes = (uint32_t)qb_encoded_query_bytes(s); p.q_off = (s->kind == QB_KIND_SQ8) ? d_q_off : nullptr;
    p.nq = nq; p.top = top; p.ef = ef; p.entry = entry; p.entry_level = entry_level;
    p.deleted = s->d_deleted; p.deleted2 = d_deleted2;
    p.out = d_out; p.out_counts = d_counts; p.id_base = s->id_base; p.stats = g->d_stats;
    const bool acorn = algo == ALGO_ACORN;
    p.hop_cap = acorn ? acorn_hop_cap(g->m0) : HNSW_MAX_LINKS;
    uint32_t q_smem = p.q_bytes;
    if (custom) {
        p.ckind = custom->kind; p.n_a = custom->n_a; p.n_b = custom->n_b;
        p.n_ex = custom->n_ex; p.ex_first = custom->ex_first; p.ex_stride = custom->ex_stride;
        p.coef = custom->d_coef; p.n_coef = custom->n_coef;
        p.cep = custom->d_cep; p.cep_counts = custom->d_cep_counts; p.n_cep = custom->n_cep;
        p.lo_end = g->level_offsets_ext.empty() ? 0 : g->level_offsets_ext.back();
        p.stats = g->d_stats + 2 * custom->stats_slot;
        if (custom->internal_out) p.id_base = 0;
        // the examples are staged in shared memory when they fit in HNSW_CUSTOM_SMEM, which keeps several queries in flight per SM;
        // larger sets are read from global memory (L1 / L2) by the same chains
        const uint64_t ex_bytes = (uint64_t)p.n_ex * p.q_bytes;
        p.ex_smem = ex_bytes <= HNSW_CUSTOM_SMEM ? 1u : 0u;
        q_smem = p.ex_smem ? (uint32_t)ex_bytes : 0u;
        p.q_smem = q_smem;
    }
    if (mv_custom) {
        // multivector examples: points and filter as for a MaxSim query; all of a query's example vectors are staged in shared memory
        // when the largest query's fit in HNSW_CUSTOM_SMEM
        p.deleted = nullptr; p.id_base = 0;
        p.ex_smem = (uint64_t)maxsim->max_q * p.q_bytes <= HNSW_CUSTOM_SMEM ? 1u : 0u;
        q_smem = p.ex_smem ? maxsim->max_q * p.q_bytes : 0u;
        p.q_smem = q_smem;
        p.stats = g->d_stats + 8;
    } else if (maxsim) {
        // points are numbered 0 .. n_points - 1 and filtered by the per-call bitmap over points only: the token storage's resident flags
        // are per token row
        p.deleted = nullptr; p.id_base = 0;
        mv_tok(p) = g->d_mv_tok; mv_qoff(p) = maxsim->d_qoff; mv_nv(p) = maxsim->n_vectors;
        // a query's vectors are staged in shared memory when the largest query's fit in HNSW_CUSTOM_SMEM, as custom examples are
        mv_stage_q(p) = (uint64_t)maxsim->max_q * p.q_bytes <= HNSW_CUSTOM_SMEM ? maxsim->max_q : 0u;
        q_smem = mv_stage_q(p) * p.q_bytes;
        p.q_smem = q_smem;
        p.stats = g->d_stats + 8;
    }
    const size_t smem = acorn ? acorn_smem_bytes(q_smem, ef, p.hop_cap) : hnsw_smem_bytes(q_smem, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "hnsw_search: query (%u B) + ef %u need %zu B of shared memory", q_smem, ef, smem);
    // threads per CTA: 256 = one 8-lane group per level-0 link (m0 = 32), fewer queries in flight per SM; 128 (default) = two scoring rounds
    // per hop, twice the resident queries.  The traversal is a chain of dependent memory round trips, so queries in flight is what hides them.
    // Custom and MaxSim queries are instantiated for 128 threads only.
    const int nt = (custom || maxsim) ? 128 : (qb_opt().hnsw_threads == 256 ? 256 : (qb_opt().hnsw_threads == 64 ? 64 : 128));
    int per_sm = 1;
    if (mv_custom) QB_TRY(qb_hnsw_mv_custom_launch(&p, g->d_mv_tok, maxsim->d_qoff, kind, metric, algo, 0, smem, stream, &per_sm));
    else per_sm = maxsim ? (acorn ? occupancy_dispatch<128, ALGO_ACORN, HC_MAXSIM>(kind, metric, smem) : occupancy_dispatch<128, ALGO_HNSW, HC_MAXSIM>(kind, metric, smem))
                       : custom ? (acorn ? occupancy_dispatch<128, ALGO_ACORN, 1>(kind, metric, smem) : occupancy_dispatch<128, ALGO_HNSW, 1>(kind, metric, smem))
                                : (acorn ? occupancy_nt<ALGO_ACORN>(nt, kind, metric, smem) : occupancy_nt<ALGO_HNSW>(nt, kind, metric, smem));
    p.prefetch = qb_opt().hnsw_no_prefetch ? 0 : 1;
    const unsigned max_grid = (unsigned)s->sm_count * (unsigned)per_sm;
    const unsigned grid = std::min<unsigned>(max_grid, nq);
    // per-CTA visited bitmaps + logs (grown on demand, zeroed once: the kernel leaves them clean)
    const uint64_t words = ceil_div_u64(g->n_points, 32);
    if (g->visited_slots < grid || g->visited_words != words) {
        cudaFree(g->d_visited); cudaFree(g->d_vlog); g->d_visited = nullptr; g->d_vlog = nullptr; g->visited_slots = 0;
        g->vlog_cap = 32768;
        QB_CUDA(cudaMalloc(&g->d_visited, std::max<size_t>((size_t)max_grid * words * 4, 256)));
        QB_CUDA(cudaMalloc(&g->d_vlog, (size_t)max_grid * g->vlog_cap * 4));
        QB_CUDA(cudaMemsetAsync(g->d_visited, 0, std::max<size_t>((size_t)max_grid * words * 4, 256), stream));
        g->visited_slots = max_grid; g->visited_words = words;
    }
    p.visited = g->d_visited; p.visited_words = words; p.vlog = g->d_vlog; p.vlog_cap = g->vlog_cap; p.work = g->d_work;
    QB_CUDA(cudaMemsetAsync(g->d_work, 0, 4, stream));
    if (mv_custom) return qb_hnsw_mv_custom_launch(&p, g->d_mv_tok, maxsim->d_qoff, kind, metric, algo, grid, smem, stream, nullptr);
    if (maxsim)
        return acorn ? launch_dispatch<128, ALGO_ACORN, HC_MAXSIM>(kind, metric, p, grid, smem, stream)
                     : launch_dispatch<128, ALGO_HNSW, HC_MAXSIM>(kind, metric, p, grid, smem, stream);
    if (custom)
        return acorn ? launch_dispatch<128, ALGO_ACORN, 1>(kind, metric, p, grid, smem, stream) : launch_dispatch<128, ALGO_HNSW, 1>(kind, metric, p, grid, smem, stream);
    return acorn ? launch_nt<ALGO_ACORN>(nt, kind, metric, p, grid, smem, stream) : launch_nt<ALGO_HNSW>(nt, kind, metric, p, grid, smem, stream);
}

qb_status qb_hnsw_read_stats(qb_hnsw* g, cudaStream_t stream, uint64_t* evals_by_slot) {
    unsigned long long h[12] = {};
    QB_CUDA(cudaMemcpyAsync(h, g->d_stats, sizeof(h), cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    QB_CUDA(cudaMemsetAsync(g->d_stats, 0, sizeof(h), stream));
    g->hops += h[0] + h[2] + h[4] + h[8]; g->evals += h[1] + h[3] + h[5] + h[9]; g->base_evals += h[6];
    g->mv_rows += h[10]; g->mv_qrows += h[11];
    if (evals_by_slot) { evals_by_slot[0] = h[1]; evals_by_slot[1] = h[3]; }
    return QB_OK;
}
