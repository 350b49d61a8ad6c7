// qb_encode.cu — the quantizers' ENCODE step on the device (SURVEY §8f rank 2: the data format right before the path).
//
// A collection is quantized once per segment build; the reference does it row by row on CPU threads.  These kernels take
// f32 rows already resident in HBM and write the reference's row formats, bit for bit, so that the output can be handed
// to qb_storage_create_{sq8,pq,bq} (or written to the segment's quantized.data file) without a round trip through the host:
//   SQ8  EncodedVectorsU8::encode          lib/quantization/src/encoded_vectors_u8.rs:143-316  (quantile = None: :194-208 skipped)
//        row = [f32 v_off][actual_dim x u8], encode_value :95-98, offsets :256-276, get_shift :116-134
//   BQ   EncodedVectorsBin::encode_vector  encoded_vectors_binary.rs:531-671  (one bit / two bits / one-and-a-half bits)
//   PQ   EncodedVectorsPQ::encode_vector   encoded_vectors_pq.rs:301-329     (argmin of the squared L2 to 256 centroids per chunk,
//        first minimum wins, sequential unfused f32 sums)
// Quantizer TRAINING (quantiles, k-means) stays with the caller: the reference's own training is RNG-dependent (SURVEY §8c).
#include "qb_internal.h"

namespace {

// ---------------------------------------------------------------------------------------------- SQ8
__device__ __forceinline__ uint32_t sq8_value(float v, float offset, float alpha) {  // encoded_vectors_u8.rs:95-98
    float i = __fdiv_rn(__fsub_rn(v, offset), alpha);
    if (i < 0.0f) i = 0.0f;       // f32::clamp keeps NaN
    if (i > 127.0f) i = 127.0f;
    const float r = roundf(i);    // f32::round: half away from zero
    return (r != r) ? 0u : (uint32_t)r;  // NaN as u8 = 0
}

// one warp per row; lane l encodes elements 4l .. 4l+3 of every 128-element block and stores them as one u32
__global__ void __launch_bounds__(256) sq8_encode_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint32_t ad, uint64_t count, float alpha,
                                                              float offset, int is_dot, int is_l1, int invert, float shift, uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    const uint32_t pad = sq8_value(is_dot ? 0.0f : offset, offset, alpha);  // placeholder of the alignment tail, :240-254
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < count; r += warps) {
        const float* src = rows + r * stride_f;
        uint8_t* dst = out + r * (uint64_t)(4 + ad);
        uint32_t sum = 0, sum2 = 0;
        for (uint32_t b = (uint32_t)lane * 4; b < ad; b += 128) {
            uint32_t word = 0;
#pragma unroll
            for (uint32_t k = 0; k < 4; ++k) {
                const uint32_t i = b + k;
                const uint32_t c = (i < dim) ? sq8_value(src[i], offset, alpha) : pad;
                word |= c << (8 * k);
                sum += c;
                sum2 += c * c;
            }
            *reinterpret_cast<uint32_t*>(dst + 4 + b) = word;  // rows are 4 + 16k bytes: 4-byte aligned
        }
        // the reference folds `code as f32` sequentially; every partial sum is an integer, so while the total stays below 2^24
        // the f32 fold equals the integer sum (the launcher sends larger rows to the sequential kernel below)
        for (int o = 16; o > 0; o >>= 1) { sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o); sum2 += __shfl_xor_sync(0xFFFFFFFFu, sum2, o); }
        if (lane == 0) {
            float off;
            if (is_dot) off = __fmul_rn(__fmul_rn((float)sum, alpha), offset);        // :256-262
            else if (is_l1) off = 0.0f;
            else off = __fmul_rn(__fmul_rn((float)sum2, alpha), alpha);              // :268-274
            if (invert) off = -off;
            *reinterpret_cast<float*>(dst) = __fadd_rn(shift, off);                   // get_shift + offset, :276-283
        }
    }
}

// rows whose code sums can leave the f32-exact window (L2 with actual_dim > 1040): thread 0 folds in the reference's order
__global__ void __launch_bounds__(256) sq8_encode_rows_seq_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint32_t ad, uint64_t count,
                                                                  float alpha, float offset, int is_dot, int is_l1, int invert, float shift,
                                                                  uint8_t* __restrict__ out) {
    const uint32_t pad = sq8_value(is_dot ? 0.0f : offset, offset, alpha);
    for (uint64_t r = blockIdx.x; r < count; r += gridDim.x) {
        const float* src = rows + r * stride_f;
        uint8_t* dst = out + r * (uint64_t)(4 + ad);
        for (uint32_t i = threadIdx.x; i < ad; i += blockDim.x) dst[4 + i] = (uint8_t)((i < dim) ? sq8_value(src[i], offset, alpha) : pad);
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = -0.0f;
            if (is_dot) { for (uint32_t i = 0; i < ad; ++i) s = __fadd_rn(s, (float)dst[4 + i]); s = __fmul_rn(__fmul_rn(s, alpha), offset); }
            else if (is_l1) s = 0.0f;
            else { for (uint32_t i = 0; i < ad; ++i) { const float c = (float)dst[4 + i]; s = __fadd_rn(s, __fmul_rn(c, c)); } s = __fmul_rn(__fmul_rn(s, alpha), alpha); }
            if (invert) s = -s;
            *reinterpret_cast<float*>(dst) = __fadd_rn(shift, s);
        }
        __syncthreads();
    }
}

// global min / max of all values (quantile.rs find_min_max_from_iter: plain comparisons, NaN never wins)
__global__ void __launch_bounds__(256) minmax_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t count, float* __restrict__ partial) {
    float mn = 3.402823466e+38f, mx = -3.402823466e+38f;
    const uint64_t total = count * (uint64_t)dim;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const float v = rows[(i / dim) * stride_f + (i % dim)];
        if (v < mn) mn = v;
        if (v > mx) mx = v;
    }
    __shared__ float s_mn[8], s_mx[8];
    for (int o = 16; o > 0; o >>= 1) {
        const float a = __shfl_xor_sync(0xFFFFFFFFu, mn, o), b = __shfl_xor_sync(0xFFFFFFFFu, mx, o);
        if (a < mn) mn = a;
        if (b > mx) mx = b;
    }
    if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) { if (s_mn[w] < mn) mn = s_mn[w]; if (s_mx[w] > mx) mx = s_mx[w]; }
        partial[2 * blockIdx.x] = mn;
        partial[2 * blockIdx.x + 1] = mx;
    }
}

// ---------------------------------------------------------------------------------------------- BQ
// encode_two_bits_value, encoded_vectors_binary.rs:636-671: bit 0 of the result = first bit, bit 1 = second bit
__device__ __forceinline__ uint32_t bq_two_bits(float value, const float* __restrict__ mean_std, uint32_t i) {
    if (!mean_std) return value > 0.0f ? 3u : 0u;
    const float mean = mean_std[2 * i], sd = mean_std[2 * i + 1];
    if (sd < 1.1920929e-7f) return value > 0.0f ? 1u : 0u;
    const float vz = __fdiv_rn(__fsub_rn(value, mean), sd);
    const float SIGMAS = __fdiv_rn(2.0f, 3.0f);
    if (vz <= -SIGMAS) return 0u;
    if (vz < SIGMAS) return 1u;
    return 3u;
}

// one warp per 32-bit word of a row: lane k decides bit p = 32 w + k, a ballot assembles the word (little-endian bit order
// over the row = bit (i % 128) of u128 word i / 128)
__global__ void __launch_bounds__(256) bq_encode_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t count, int encoding,
                                                             const float* __restrict__ mean_std, uint32_t row_bytes, uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint32_t words = row_bytes >> 2;
    const uint64_t total = count * (uint64_t)words;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t g = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < total; g += warps) {
        const uint64_t r = g / words;
        const uint32_t w = (uint32_t)(g % words);
        const float* src = rows + r * stride_f;
        const uint64_t p = (uint64_t)w * 32 + lane;
        bool bit = false;
        if (p < dim) {
            const uint32_t i = (uint32_t)p;
            bit = (encoding == QB_BQ_ONE_BIT) ? (src[i] > 0.0f) : ((bq_two_bits(src[i], mean_std, i) & 1u) != 0);
        } else if (encoding == QB_BQ_TWO_BITS && p < 2ull * dim) {
            const uint32_t i = (uint32_t)(p - dim);
            bit = (bq_two_bits(src[i], mean_std, i) & 2u) != 0;
        } else if (encoding == QB_BQ_ONE_AND_HALF_BITS && p < (uint64_t)dim + (dim + 1) / 2) {
            const uint32_t i = 2 * (uint32_t)(p - dim);  // two neighbouring coordinates share their second bit (:608-634)
            bit = (bq_two_bits(src[i], mean_std, i) & 2u) != 0;
            if (i + 1 < dim) bit = bit || ((bq_two_bits(src[i + 1], mean_std, i + 1) & 2u) != 0);
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (lane == 0) reinterpret_cast<uint32_t*>(out + r * (uint64_t)row_bytes)[w] = word;
    }
}

// ---------------------------------------------------------------------------------------------- PQ
// block = (chunk j, tile of rows): the 256 centroid sub-vectors of chunk j sit in shared memory (every thread reads the same
// element at the same time: a broadcast), one thread per row keeps its sub-vector in registers
constexpr int PQ_MAX_SUB = 64;
template <int SUB>  // SUB >= chunk: register sub-vector size (8, 16, 32 or 64)
__global__ void __launch_bounds__(256) pq_encode_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint32_t chunk, uint32_t m,
                                                             const float* __restrict__ centroids, uint32_t n_centroids, uint64_t count, uint8_t* __restrict__ codes) {
    extern __shared__ float cs[];  // [n_centroids][len]
    const uint32_t j = blockIdx.y;
    const uint32_t s = j * chunk, e = min(s + chunk, dim), len = e - s;
    for (uint32_t i = threadIdx.x; i < n_centroids * len; i += blockDim.x) cs[i] = centroids[(uint64_t)(i / len) * dim + s + (i % len)];
    __syncthreads();
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < count; r += (uint64_t)gridDim.x * blockDim.x) {
        const float* src = rows + r * stride_f + s;
        float v[SUB];
#pragma unroll
        for (int k = 0; k < SUB; ++k) v[k] = (k < (int)len) ? src[k] : 0.0f;
        float min_d = 3.402823466e+38f;
        uint32_t min_c = 0;
        for (uint32_t c = 0; c < n_centroids; ++c) {
            const float* cd = cs + c * len;
            float d = -0.0f;  // Iterator::sum::<f32>() starts from -0.0
#pragma unroll
            for (int k = 0; k < SUB; ++k)
                if (k < (int)len) { const float t = __fsub_rn(v[k], cd[k]); d = __fadd_rn(d, __fmul_rn(t, t)); }
            if (d < min_d) { min_d = d; min_c = c; }  // first minimum wins (:318-326)
        }
        codes[r * (uint64_t)m + j] = (uint8_t)min_c;
    }
}

}  // namespace

static qb_status use_dev(int device) {
    QB_CUDA(cudaSetDevice(device));
    return QB_OK;
}

extern "C" qb_status qb_sq8_find_alpha_offset_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, float* alpha,
                                                     float* offset) {
    QB_CHECK(dev_rows && alpha && offset && dim >= 1 && count >= 1, QB_ERR_INVALID, "sq8_find_alpha_offset: bad arguments");
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0 && row_stride_bytes >= (uint64_t)dim * 4, QB_ERR_INVALID, "sq8_find_alpha_offset: bad row stride");
    QB_TRY(use_dev(device));
    const unsigned grid = 132 * 8;
    float* d_part = nullptr;
    QB_CUDA(cudaMalloc(&d_part, grid * 2 * sizeof(float)));
    minmax_kernel<<<grid, 256>>>(dev_rows, row_stride_bytes / 4, dim, count, d_part);
    QB_LAUNCHED();
    std::vector<float> h(grid * 2);
    cudaError_t e = cudaMemcpy(h.data(), d_part, h.size() * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(d_part);
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "sq8_find_alpha_offset: %s", cudaGetErrorString(e));
    float mn = h[0], mx = h[1];
    for (unsigned i = 1; i < grid; ++i) { if (h[2 * i] < mn) mn = h[2 * i]; if (h[2 * i + 1] > mx) mx = h[2 * i + 1]; }
    volatile float range = mx - mn;            // alpha = (max - min) / 127, offset = min (encoded_vectors_u8.rs:523-527)
    *alpha = range / 127.0f;
    *offset = mn;
    return QB_OK;
}

extern "C" qb_status qb_sq8_encode_rows_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, float alpha, float offset,
                                               qb_qdistance dt, int invert, uint8_t* dev_out, void* stream) {
    QB_CHECK(dev_rows && dev_out && dim >= 1, QB_ERR_INVALID, "sq8_encode_rows: bad arguments");
    if (count == 0) return QB_OK;
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0 && row_stride_bytes >= (uint64_t)dim * 4, QB_ERR_INVALID, "sq8_encode_rows: bad row stride");
    QB_TRY(use_dev(device));
    const uint32_t ad = dim + (16 - dim % 16) % 16;
    const int is_dot = (dt == QB_QD_DOT || dt == QB_QD_COSINE), is_l1 = (dt == QB_QD_L1);
    float shift = 0.0f;
    if (is_dot) { volatile float a = (float)ad * offset; shift = a * offset; }  // get_shift, :116-134
    if (invert) shift = -shift;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool exact_window = is_dot ? ((uint64_t)ad * 127ull < (1ull << 24)) : (is_l1 || (uint64_t)ad * 127ull * 127ull < (1ull << 24));
    if (exact_window) {
        const unsigned grid = (unsigned)std::min<uint64_t>(ceil_div_u64(count, 8), 132ull * 32);
        sq8_encode_rows_kernel<<<grid, 256, 0, st>>>(dev_rows, row_stride_bytes / 4, dim, ad, count, alpha, offset, is_dot, is_l1, invert, shift, dev_out);
    } else {
        const unsigned grid = (unsigned)std::min<uint64_t>(count, 132ull * 32);
        sq8_encode_rows_seq_kernel<<<grid, 256, 0, st>>>(dev_rows, row_stride_bytes / 4, dim, ad, count, alpha, offset, is_dot, is_l1, invert, shift, dev_out);
    }
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

extern "C" uint32_t qb_bq_row_bytes(uint32_t dim, qb_bq_encoding encoding) {  // get_quantized_vector_size_from_params, encoded_vectors_binary.rs:829-839
    uint64_t ext = dim;
    if (encoding == QB_BQ_TWO_BITS) ext = (uint64_t)dim * 2;
    else if (encoding == QB_BQ_ONE_AND_HALF_BITS) ext = ((uint64_t)dim * 3 + 1) / 2;
    if (ext < 1) ext = 1;
    return (uint32_t)(((ext + 127) / 128) * 16);
}

extern "C" qb_status qb_bq_encode_rows_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, qb_bq_encoding encoding,
                                              const float* mean_std, uint8_t* dev_out, void* stream) {
    QB_CHECK(dev_rows && dev_out && dim >= 1, QB_ERR_INVALID, "bq_encode_rows: bad arguments");
    QB_CHECK(encoding >= QB_BQ_ONE_BIT && encoding <= QB_BQ_ONE_AND_HALF_BITS, QB_ERR_INVALID, "bq_encode_rows: unknown encoding");
    if (count == 0) return QB_OK;
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0 && row_stride_bytes >= (uint64_t)dim * 4, QB_ERR_INVALID, "bq_encode_rows: bad row stride");
    QB_TRY(use_dev(device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    float* d_ms = nullptr;
    if (mean_std && encoding != QB_BQ_ONE_BIT) {
        QB_CUDA(cudaMalloc(&d_ms, (size_t)dim * 2 * sizeof(float)));
        cudaError_t e = cudaMemcpyAsync(d_ms, mean_std, (size_t)dim * 2 * sizeof(float), cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { cudaFree(d_ms); qb_set_error("bq_encode_rows: %s", cudaGetErrorString(e)); return QB_ERR_CUDA; }
    }
    const uint32_t row_bytes = qb_bq_row_bytes(dim, encoding);
    const uint64_t total_words = count * (uint64_t)(row_bytes / 4);
    const unsigned grid = (unsigned)std::min<uint64_t>(ceil_div_u64(total_words, 8), 132ull * 32);
    bq_encode_rows_kernel<<<grid, 256, 0, st>>>(dev_rows, row_stride_bytes / 4, dim, count, (int)encoding, d_ms, row_bytes, dev_out);
    QB_LAUNCHED();
    cudaError_t e = cudaGetLastError();
    if (d_ms) { cudaStreamSynchronize(st); cudaFree(d_ms); }
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "bq_encode_rows: %s", cudaGetErrorString(e));
    return QB_OK;
}

extern "C" qb_status qb_pq_encode_rows_device(int32_t device, uint32_t dim, uint32_t chunk, uint32_t n_centroids, const float* centroids, uint64_t count,
                                              const float* dev_rows, uint64_t row_stride_bytes, uint8_t* dev_codes, void* stream) {
    QB_CHECK(dev_rows && dev_codes && centroids && dim >= 1 && chunk >= 1, QB_ERR_INVALID, "pq_encode_rows: bad arguments");
    QB_CHECK(n_centroids >= 1 && n_centroids <= 256, QB_ERR_INVALID, "pq_encode_rows: %u centroids (codes are one byte)", n_centroids);
    QB_CHECK(chunk <= (uint32_t)PQ_MAX_SUB, QB_ERR_UNSUPPORTED, "pq_encode_rows: chunk size %u > %d", chunk, PQ_MAX_SUB);
    if (count == 0) return QB_OK;
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0 && row_stride_bytes >= (uint64_t)dim * 4, QB_ERR_INVALID, "pq_encode_rows: bad row stride");
    QB_TRY(use_dev(device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const uint32_t m = (dim + chunk - 1) / chunk;  // get_vector_division, encoded_vectors_pq.rs:164-169
    float* d_c = nullptr;
    QB_CUDA(cudaMalloc(&d_c, (size_t)n_centroids * dim * sizeof(float)));
    cudaError_t e = cudaMemcpyAsync(d_c, centroids, (size_t)n_centroids * dim * sizeof(float), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        const size_t smem = (size_t)n_centroids * chunk * sizeof(float);  // <= 64 KB
        const unsigned gx = (unsigned)std::min<uint64_t>(ceil_div_u64(count, 256), 132ull * 4);
        auto launch = [&](auto kernel) {
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return;
            kernel<<<dim3(gx, m), 256, smem, st>>>(dev_rows, row_stride_bytes / 4, dim, chunk, m, d_c, n_centroids, count, dev_codes);
            QB_LAUNCHED();
            e = cudaGetLastError();
        };
        if (chunk <= 8) launch(pq_encode_rows_kernel<8>);
        else if (chunk <= 16) launch(pq_encode_rows_kernel<16>);
        else if (chunk <= 32) launch(pq_encode_rows_kernel<32>);
        else launch(pq_encode_rows_kernel<64>);
    }
    cudaStreamSynchronize(st);
    cudaFree(d_c);
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "pq_encode_rows: %s", cudaGetErrorString(e));
    return QB_OK;
}
