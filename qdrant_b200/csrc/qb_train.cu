// qb_train.cu — quantizer TRAINING on the device (SURVEY §8f rank 2, the half that precedes qb_*_encode_rows_device).
//
//   BQ   VectorStats::build                     lib/quantization/src/vector_stats.rs:48-117   per-coordinate Welford mean / stddev in f64
//   SQ8  find_quantile_interval                 lib/quantization/src/quantile.rs:35-88        (min, max) of the values between two order
//        + alpha_offset_from_min_max            encoded_vectors_u8.rs:523-527                 statistics of the sampled values
//   PQ   find_centroids -> kmeans               encoded_vectors_pq.rs:342-407, kmeans.rs:9-167 Lloyd iterations per chunk: first-minimum
//                                                                                             assignment, f64 means, L1 centroid shift < accuracy
//
// What is deterministic in the reference is reproduced operation for operation (the Welford recurrences, the order statistics, the
// per-thread-range f64 partial sums of update_centroids merged in thread order, the sequential f32 distance sums).  What the reference
// draws from an unseeded RNG is an INPUT here: the caller passes the sampled vectors (Permutor-sampled rows in the reference,
// quantile.rs:286-314, encoded_vectors_pq.rs:365-372) and a seed for the re-seeding of empty k-means clusters (kmeans.rs:115 uses
// rand::rng()); the CPU restatement used by the tests follows the same rule, so training parity is pinned given (sample, seed, thread count).
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>

#include "qb_internal.h"

namespace {

// ---------------------------------------------------------------- BQ: per-coordinate Welford (one thread per coordinate, rows in order)
__global__ void bq_stats_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t count, float* __restrict__ mean_std, float* __restrict__ min_max) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= dim) return;
    double mean = 0.0, m2 = 0.0;
    float mn = 3.402823466e+38f, mx = -3.402823466e+38f;
    for (uint64_t i = 0; i < count; ++i) {
        const float v = rows[i * stride_f + k];
        if (v < mn) mn = v;
        if (v > mx) mx = v;
        const double x = (double)v, cnt = (double)(i + 1);
        const double delta = __dsub_rn(x, mean);
        mean = __dadd_rn(mean, __ddiv_rn(delta, cnt));
        m2 = __dadd_rn(m2, __dmul_rn(delta, __dsub_rn(x, mean)));
    }
    mean_std[2 * k] = (float)mean;
    mean_std[2 * k + 1] = count > 1 ? (float)__dsqrt_rn(__ddiv_rn(m2, (double)(count - 1))) : 0.0f;
    if (min_max) { min_max[2 * k] = mn; min_max[2 * k + 1] = mx; }
}

// ---------------------------------------------------------------- SQ8 quantile: orderable keys for a total order of the sampled values
__global__ void f32_to_sort_keys(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t n, uint32_t* __restrict__ keys) {
    const uint64_t total = n * dim;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t u = __float_as_uint(rows[(i / dim) * stride_f + (i % dim)]);
        keys[i] = (u & 0x80000000u) ? ~u : (u | 0x80000000u);     // ascending u32 order == ascending float order (partial_cmp on non-NaN values)
    }
}

// ---------------------------------------------------------------- PQ k-means
struct KmParams {
    const float* sample; uint64_t stride_f; uint32_t n, dim, m, K;     // n sampled vectors; m chunks; K centroids
    const uint32_t* div;                                               // [m][2]
    float* cent;            // [m][K][clen_max]  current centroids per chunk (chunk-local layout)
    float* cent_new;        // same
    uint32_t* idx;          // [m][n]
    uint32_t clen_max;
    uint32_t groups;        // the reference's max_threads: f64 partial sums per contiguous range of samples, merged in range order
    uint32_t* converged;    // [m]
    uint32_t iter; unsigned long long seed;
    float accuracy;
};

// update_indexes (kmeans.rs:136-167): first strict minimum of the sequential f32 sum of (a - b)^2, centroids of the chunk in shared memory
__global__ void __launch_bounds__(256) km_assign_kernel(const KmParams p) {
    extern __shared__ float c_s[];
    const uint32_t j = blockIdx.y;
    if (p.converged[j]) return;
    const uint32_t s = p.div[2 * j], clen = p.div[2 * j + 1] - s;
    const float* cj = p.cent + (size_t)j * p.K * p.clen_max;
    for (uint32_t i = threadIdx.x; i < p.K * clen; i += blockDim.x) c_s[i] = cj[(size_t)(i / clen) * p.clen_max + (i % clen)];
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
        const float* v = p.sample + (uint64_t)i * p.stride_f + s;
        float best = 3.402823466e+38f;
        uint32_t bi = 0;
        for (uint32_t c = 0; c < p.K; ++c) {
            float acc = -0.0f;                                   // f32 Sum folds from -0.0
            for (uint32_t k = 0; k < clen; ++k) { const float d = __fsub_rn(v[k], c_s[c * clen + k]); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
            if (acc < best) { best = acc; bi = c; }
        }
        p.idx[(size_t)j * p.n + i] = bi;
    }
}

__device__ __forceinline__ unsigned long long km_mix(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}

// update_centroids (kmeans.rs:49-134): one thread per (chunk, centroid, coordinate); per sample range (the reference's thread ranges:
// chunk_size = n / groups, the last range takes the remainder) a sequential f64 sum, ranges added in order, mean = sum / count (f64), cast to f32
__global__ void __launch_bounds__(256) km_update_kernel(const KmParams p) {
    const uint32_t j = blockIdx.y;
    if (p.converged[j]) return;
    const uint32_t s = p.div[2 * j], clen = p.div[2 * j + 1] - s;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.K * clen) return;
    const uint32_t c = t / clen, k = t % clen;
    const uint32_t* idx = p.idx + (size_t)j * p.n;
    const uint32_t chunk = p.n / p.groups;
    double total = 0.0;
    unsigned long long cnt = 0;
    for (uint32_t g = 0; g < p.groups; ++g) {
        const uint32_t b = chunk * g, e = (g + 1 == p.groups) ? p.n : chunk * (g + 1);
        double part = 0.0;
        for (uint32_t i = b; i < e; ++i)
            if (idx[i] == c) { part = __dadd_rn(part, (double)p.sample[(uint64_t)i * p.stride_f + s + k]); ++cnt; }
        total = __dadd_rn(total, part);
    }
    float out;
    if (cnt == 0) {
        // empty cluster: the reference re-seeds it with a random sampled vector (rand::rng(), kmeans.rs:113-121); here the index is a
        // function of (seed, iteration, chunk, centroid) so that a CPU restatement can follow
        const uint32_t di = (uint32_t)(km_mix(p.seed ^ km_mix(((unsigned long long)p.iter << 40) ^ ((unsigned long long)j << 20) ^ c)) % p.n);
        out = (float)(double)p.sample[(uint64_t)di * p.stride_f + s + k];
    } else {
        out = (float)__ddiv_rn(total, (double)cnt);
    }
    p.cent_new[((size_t)j * p.K + c) * p.clen_max + k] = out;
}

// diff = sum over centroid coordinates, in order, of |old - new| (f32, from -0.0); converged when diff < accuracy; old = new either way
__global__ void km_diff_kernel(const KmParams p) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.m || p.converged[j]) return;
    const uint32_t clen = p.div[2 * j + 1] - p.div[2 * j];
    float* co = p.cent + (size_t)j * p.K * p.clen_max;
    const float* cn = p.cent_new + (size_t)j * p.K * p.clen_max;
    float diff = -0.0f;
    for (uint32_t c = 0; c < p.K; ++c)
        for (uint32_t k = 0; k < clen; ++k) {
            const size_t o = (size_t)c * p.clen_max + k;
            diff = __fadd_rn(diff, fabsf(__fsub_rn(co[o], cn[o])));
            co[o] = cn[o];
        }
    if (diff < p.accuracy) p.converged[j] = 1u;
}

__global__ void km_init_kernel(const KmParams p) {   // initial centroids = the first K sampled vectors (kmeans.rs:28)
    const uint32_t j = blockIdx.y;
    const uint32_t s = p.div[2 * j], clen = p.div[2 * j + 1] - s;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < p.K * clen; t += gridDim.x * blockDim.x)
        p.cent[((size_t)j * p.K + t / clen) * p.clen_max + (t % clen)] = p.sample[(uint64_t)(t / clen) * p.stride_f + s + (t % clen)];
}

}  // namespace

static qb_status train_use_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); qb_set_error("no CUDA device (this library has no CPU fallback)"); return QB_ERR_NO_DEVICE; }
    QB_CHECK(device >= 0 && device < n, QB_ERR_INVALID, "device %d out of range", device);
    QB_CUDA(cudaSetDevice(device));
    return QB_OK;
}

extern "C" qb_status qb_bq_vector_stats_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, float* mean_std_out,
                                               float* min_max_out) {
    QB_CHECK(dev_rows && mean_std_out && dim >= 1, QB_ERR_INVALID, "bq_vector_stats: bad arguments");
    QB_TRY(train_use_device(device));
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0, QB_ERR_INVALID, "bq_vector_stats: stride must be a multiple of 4");
    float* d = nullptr;
    QB_CUDA(cudaMalloc(&d, (size_t)dim * 16));
    bq_stats_kernel<<<(dim + 63) / 64, 64>>>(dev_rows, row_stride_bytes / 4, dim, count, d, d + 2 * (size_t)dim);
    QB_LAUNCHED();
    cudaError_t e = cudaMemcpy(mean_std_out, d, (size_t)dim * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && min_max_out) e = cudaMemcpy(min_max_out, d + 2 * (size_t)dim, (size_t)dim * 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) { qb_set_error("bq_vector_stats: %s", cudaGetErrorString(e)); return QB_ERR_CUDA; }
    return QB_OK;
}

extern "C" qb_status qb_sq8_quantile_interval_device(int32_t device, uint32_t dim, uint64_t n_sample, const float* dev_sample_rows, uint64_t row_stride_bytes,
                                                     float quantile, float* alpha, float* offset, int32_t* found) {
    QB_CHECK(dev_sample_rows && alpha && offset && found && dim >= 1, QB_ERR_INVALID, "sq8_quantile_interval: bad arguments");
    *found = 0;
    QB_TRY(train_use_device(device));
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    const uint64_t len = n_sample * dim;
    // find_quantile_interval, quantile.rs:35-88 (the caller applied `count < 127 || quantile >= 1.0 -> None` and the sampling)
    if (quantile >= 1.0f || len < 4) return QB_OK;
    uint64_t cut = std::min<uint64_t>((len - 1) / 2, (uint64_t)((float)n_sample * (1.0f - quantile) / 2.0f));
    cut = std::max<uint64_t>(cut, 1);
    // values strictly between the cut-th and the (len - cut)-th order statistic: sorted[cut + 1 .. len - cut - 1]
    if (len - cut < cut + 1 + 2) return QB_OK;      // selected_values.len() < 2
    QB_CHECK(len < (1ull << 31), QB_ERR_UNSUPPORTED, "sq8_quantile_interval: %llu sampled values", (unsigned long long)len);
    uint32_t *d_in = nullptr, *d_out = nullptr;
    void* d_tmp = nullptr;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, d_in, d_out, (int)len);
    qb_status st = QB_OK;
    if (cudaMalloc(&d_in, len * 4) != cudaSuccess || cudaMalloc(&d_out, len * 4) != cudaSuccess || cudaMalloc(&d_tmp, tmp_bytes + 256) != cudaSuccess) st = QB_ERR_OOM;
    uint32_t k2[2] = {0, 0};
    if (st == QB_OK) {
        f32_to_sort_keys<<<(unsigned)std::min<uint64_t>((len + 255) / 256, 132 * 16), 256>>>(dev_sample_rows, row_stride_bytes / 4, dim, n_sample, d_in);
        QB_LAUNCHED();
        cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, d_in, d_out, (int)len);
        cudaError_t e = cudaMemcpy(&k2[0], d_out + cut + 1, 4, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(&k2[1], d_out + (len - cut - 1), 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { qb_set_error("sq8_quantile_interval: %s", cudaGetErrorString(e)); st = QB_ERR_CUDA; }
    } else qb_set_error("sq8_quantile_interval: cudaMalloc failed");
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_tmp);
    if (st != QB_OK) return st;
    const float mn = qb_unorderable(k2[0]), mx = qb_unorderable(k2[1]);
    *alpha = (mx - mn) / 127.0f;     // alpha_offset_from_min_max, encoded_vectors_u8.rs:523-527 (host f32 arithmetic on two scalars)
    *offset = mn;
    *found = 1;
    return QB_OK;
}

extern "C" qb_status qb_pq_train_device(int32_t device, uint32_t dim, uint32_t chunk, uint32_t n_centroids, uint64_t n_sample, const float* dev_sample_rows,
                                        uint64_t row_stride_bytes, uint32_t max_iterations, float accuracy, uint32_t max_threads, uint64_t seed, float* centroids_out,
                                        uint32_t* iterations_out) {
    QB_CHECK(dev_sample_rows && centroids_out && dim >= 1 && chunk >= 1 && n_centroids >= 1 && n_centroids <= 256 && max_threads >= 1, QB_ERR_INVALID, "pq_train: bad arguments");
    QB_TRY(train_use_device(device));
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0 && n_sample < (1ull << 31), QB_ERR_INVALID, "pq_train: bad stride / sample size");
    const uint32_t m = (dim + chunk - 1) / chunk, n = (uint32_t)n_sample, K = n_centroids;
    if (iterations_out) *iterations_out = 0;
    if (n <= K) {   // find_centroids: not enough vectors -> the points themselves, the rest zeros (encoded_vectors_pq.rs:355-362)
        memset(centroids_out, 0, (size_t)K * dim * 4);
        if (n) QB_CUDA(cudaMemcpy2D(centroids_out, (size_t)dim * 4, dev_sample_rows, row_stride_bytes, (size_t)dim * 4, n, cudaMemcpyDeviceToHost));
        return QB_OK;
    }
    std::vector<uint32_t> div(2 * (size_t)m);   // get_vector_division, encoded_vectors_pq.rs:164-169
    for (uint32_t j = 0; j < m; ++j) { div[2 * j] = j * chunk; div[2 * j + 1] = std::min(dim, (j + 1) * chunk); }
    KmParams p{};
    p.sample = dev_sample_rows; p.stride_f = row_stride_bytes / 4; p.n = n; p.dim = dim; p.m = m; p.K = K; p.clen_max = chunk; p.groups = std::min(max_threads, n);
    p.accuracy = accuracy; p.seed = seed;
    const size_t cbytes = (size_t)m * K * chunk * 4;
    uint32_t* d_div = nullptr;
    qb_status st = QB_OK;
    if (cudaMalloc(&d_div, div.size() * 4) != cudaSuccess || cudaMalloc(&p.cent, cbytes) != cudaSuccess || cudaMalloc(&p.cent_new, cbytes) != cudaSuccess ||
        cudaMalloc(&p.idx, (size_t)m * n * 4) != cudaSuccess || cudaMalloc(&p.converged, (size_t)m * 4 + 256) != cudaSuccess) {
        qb_set_error("pq_train: cudaMalloc failed"); st = QB_ERR_OOM;
    }
    uint32_t iters = 0;
    if (st == QB_OK) {
        cudaMemcpy(d_div, div.data(), div.size() * 4, cudaMemcpyHostToDevice);
        p.div = d_div;
        cudaMemset(p.converged, 0, (size_t)m * 4);
        cudaMemset(p.cent, 0, cbytes); cudaMemset(p.cent_new, 0, cbytes);
        const dim3 gi((K * chunk + 255) / 256, m), ga(std::min<uint32_t>((n + 255) / 256, 64), m), gu((K * chunk + 255) / 256, m);
        km_init_kernel<<<gi, 256>>>(p);
        QB_LAUNCHED();
        std::vector<uint32_t> conv(m);
        for (uint32_t it = 0; it < max_iterations; ++it) {
            p.iter = it;
            km_assign_kernel<<<ga, 256, (size_t)K * chunk * 4>>>(p);
            km_update_kernel<<<gu, 256>>>(p);
            km_diff_kernel<<<(m + 63) / 64, 64>>>(p);
            QB_LAUNCHED(); QB_LAUNCHED(); QB_LAUNCHED();
            iters = it + 1;
            if ((it & 3) == 3 || it + 1 == max_iterations) {   // every chunk runs its own kmeans(): a converged chunk is frozen, the loop ends when all are
                if (cudaMemcpy(conv.data(), p.converged, (size_t)m * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { st = QB_ERR_CUDA; break; }
                if (std::all_of(conv.begin(), conv.end(), [](uint32_t v) { return v != 0; })) break;
            }
        }
        // Metadata.centroids: K full-dim vectors, chunk j's coordinates at [start_j, end_j) (encoded_vectors_pq.rs:399-403)
        std::vector<float> h(cbytes / 4);
        if (st == QB_OK && cudaMemcpy(h.data(), p.cent, cbytes, cudaMemcpyDeviceToHost) != cudaSuccess) st = QB_ERR_CUDA;
        if (st == QB_OK)
            for (uint32_t j = 0; j < m; ++j)
                for (uint32_t c = 0; c < K; ++c)
                    for (uint32_t k = 0; k < div[2 * j + 1] - div[2 * j]; ++k) centroids_out[(size_t)c * dim + div[2 * j] + k] = h[((size_t)j * K + c) * chunk + k];
        if (st != QB_OK) qb_set_error("pq_train: %s", cudaGetErrorString(cudaGetLastError()));
    }
    cudaFree(d_div); cudaFree(p.cent); cudaFree(p.cent_new); cudaFree(p.idx); cudaFree(p.converged);
    if (iterations_out) *iterations_out = iters;
    return st;
}
