// qb_hnsw_host.cuh — host helpers shared by the graph loaders (qb_hnsw.cu) and the graph builds (qb_hnsw_build.cuh): device scratch,
// launch grids, and the offsets / neighbours step that turns per-entry link counts into a handle's plain arrays.  The handle itself is
// made by qb_hnsw_new and completed by qb_hnsw_finish_plain (qb_hnsw.cu).
#pragma once
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "qb_hnsw_traverse.cuh"

namespace {

// device temporaries of one call, freed on every exit path once the device is idle
struct HnswScratch {
    std::vector<void*> bufs;
    cudaError_t alloc(void** p, size_t bytes) {
        *p = nullptr;
        const cudaError_t e = cudaMalloc(p, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess) bufs.push_back(*p);
        return e;
    }
    ~HnswScratch() { cudaDeviceSynchronize(); for (void* b : bufs) cudaFree(b); }
};

inline unsigned hnsw_grid(uint64_t items, uint64_t per_block, uint64_t max_blocks) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div_u64(items, per_block), max_blocks));
}

// g's plain offsets and neighbours from the link count of each of its n_off offset entries (the last count 0, so the exclusive scan ends
// on the total): the scan into d_offsets, the total read back, d_neighbors allocated for it, then fill(d_offsets, d_neighbors) launches
// the caller's kernel that writes them.  d_flag (optional): a decode's device checks, read back with the total into *flag; when one is
// set nothing is allocated or filled, and the caller refuses the file.  who / what: the error messages' prefix and stage.  On failure the
// caller destroys g.  A template, so that the scan's kernels are compiled only into the objects that run it.
template <class Fill>
qb_status hnsw_link_offsets(qb_hnsw* g, uint64_t* d_counts, uint64_t n_off, HnswScratch& tmp, const char* who, const char* what,
                            const uint32_t* d_flag, uint32_t* flag, Fill fill) {
    size_t scan_bytes = 0;
    cudaError_t ce = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_counts, g->d_offsets, (int64_t)n_off);
    void* d_scan = nullptr;
    if (ce == cudaSuccess) ce = tmp.alloc(&d_scan, scan_bytes);
    if (ce == cudaSuccess) ce = cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_counts, g->d_offsets, (int64_t)n_off);
    QB_LAUNCHED();
    uint64_t total = 0;
    if (ce == cudaSuccess && d_flag) ce = cudaMemcpy(flag, d_flag, 4, cudaMemcpyDeviceToHost);
    if (ce == cudaSuccess) ce = cudaMemcpy(&total, g->d_offsets + (n_off - 1), 8, cudaMemcpyDeviceToHost);
    if (ce != cudaSuccess) { qb_set_error("%s: %s: %s", who, what, cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    if (d_flag && *flag) return QB_OK;
    g->n_neighbors = total;
    if (cudaMalloc(&g->d_neighbors, std::max<size_t>(4 * total, 256)) != cudaSuccess) {
        qb_set_error("%s: cudaMalloc failed: %s", who, cudaGetErrorString(cudaGetLastError()));
        return QB_ERR_OOM;
    }
    fill(g->d_offsets, g->d_neighbors);
    return QB_OK;
}

}  // namespace
