// torchac_batch.cu -- section F of l3c_b200.h: coding intervals and decoder rows for many streams of the torchac
// drop-in API in one launch each.  A stream is either an explicit CDF table [n_sym][Lp] or a logistic mixture given
// as [K][n_sym] planes; its integers are those of the single-stream entry points (capi.cu: table_intervals_kernel,
// plane_intervals_kernel, repitch_kernel, plane_table_kernel).
//
// Threads map to a flat index over the concatenated work of all streams (a symbol, or 8 entries of a row), so a
// launch costs what its symbols cost, however many streams there are and however ragged.  Every block finds the
// streams of its first and last index in the offset array, and its threads search only between those two.
#include <limits.h>

#include "common.cuh"
#include "dmll_math.cuh"

namespace l3c {
namespace {

constexpr int BATCH_THREADS = 256;

// the last stream j in [lo, hi] with off[j] <= i (off ascending; an empty stream shares its offset with the next one,
// which is then the one chosen)
__device__ __forceinline__ int find_stream(const int64_t *__restrict__ off, int lo, int hi, int64_t i) {
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(off + mid) <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// streams of the block's first and last index [i0, i1]
__device__ __forceinline__ void block_streams(const int64_t *__restrict__ off, int n, int64_t i0, int64_t i1, int &lo,
                                              int &hi) {
    __shared__ int s[2];
    if (threadIdx.x == 0) s[0] = find_stream(off, 0, n - 1, i0);
    if (threadIdx.x == 32) s[1] = find_stream(off, 0, n - 1, i1);
    __syncthreads();
    lo = s[0];
    hi = s[1];
}

// iv[i] = c_low | (c_high - 1) << 16 of symbol i of the concatenation; bad[j] = min over stream j's positions whose
// symbol lies outside [0, Lp - 2] (the caller fills bad with 0xFF: no such position reads as -1)
__global__ void __launch_bounds__(BATCH_THREADS)
    batch_intervals_kernel(const l3c_code_src_t *__restrict__ src, const int64_t *__restrict__ off, int n,
                           int64_t total, uint32_t *__restrict__ iv, uint32_t *__restrict__ bad) {
    const int64_t i0 = (int64_t)blockIdx.x * BATCH_THREADS;
    int lo, hi;
    block_streams(off, n, i0, min(i0 + BATCH_THREADS, total) - 1, lo, hi);
    const int64_t i = i0 + threadIdx.x;
    if (i >= total) return;
    const int j = find_stream(off, lo, hi, i);
    const l3c_code_src_t &d = src[j];
    const int64_t r = i - __ldg(off + j);
    const int Lp = d.Lp;
    const int s = d.sym[r];
    if (s < 0 || s > Lp - 2) {
        atomicMin(bad + j, (uint32_t)r);
        iv[i] = 0u;
        return;
    }
    uint32_t c_lo, c_hi;
    if (d.table) {                      // table_intervals_kernel
        c_lo = d.table[r * Lp + s];
        c_hi = (s == Lp - 2) ? 0x10000u : (uint32_t)d.table[r * Lp + s + 1];
    } else {                            // plane_intervals_kernel
        const float scale = (float)(65536 - (Lp - 1));
        c_lo = plane_cdf_u16(d.means, d.log_scales, d.probs, d.K, d.n_sym, r, d.targets[s], scale, s);
        c_hi = (s == Lp - 2) ? 0x10000u
                             : plane_cdf_u16(d.means, d.log_scales, d.probs, d.K, d.n_sym, r, d.targets[s + 1], scale,
                                             s + 1);
    }
    iv[i] = c_lo | ((c_hi - 1u) << 16);
}

// 8 entries [e0, e0 + 8) of the decoder row of symbol `row`: entries 0..L-1 of the CDF, zeros past L
__global__ void __launch_bounds__(BATCH_THREADS)
    batch_rows_kernel(const l3c_code_src_t *__restrict__ src, const int64_t *__restrict__ off, int n, int64_t total_vec,
                      uint32_t first, uint16_t *__restrict__ rows) {
    const int64_t v0 = (int64_t)blockIdx.x * BATCH_THREADS;
    int lo, hi;
    block_streams(off, n, 8 * v0, 8 * (min(v0 + BATCH_THREADS, total_vec) - 1), lo, hi);
    const int64_t v = v0 + threadIdx.x;
    if (v >= total_vec) return;
    const int j = find_stream(off, lo, hi, 8 * v);
    const l3c_code_src_t &d = src[j];
    const int64_t local = 8 * v - __ldg(off + j);
    const int L = d.Lp - 1;
    const int pitch = decode_pitch(L);
    const int64_t row = (int64_t)first + local / pitch;
    const int e0 = (int)(local % pitch);
    uint32_t w[4];
    if (d.table) {                      // repitch_kernel
        const uint16_t *t = d.table + row * d.Lp;
#pragma unroll
        for (int q = 0; q < 8; q += 2) {
            const uint32_t a = (e0 + q < L) ? (uint32_t)t[e0 + q] : 0u;
            const uint32_t b = (e0 + q + 1 < L) ? (uint32_t)t[e0 + q + 1] : 0u;
            w[q / 2] = a | (b << 16);
        }
    } else {                            // plane_table_kernel: plane_cdf_u16 for 8 targets, the K terms in order
        float tg[8], acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            tg[q] = d.targets[min(e0 + q, L - 1)];
            acc[q] = 0.f;
        }
        const int64_t N = d.n_sym;
        for (int k = 0; k < d.K; ++k) {
            const float is = __fmul_rn(expf(-d.log_scales[k * N + row]), NEG_LOG2E);
            const float mu = d.means[k * N + row];
            const float pi = d.probs[k * N + row];
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = mixture_term(acc[q], pi, __fmul_rn(__fsub_rn(tg[q], mu), is));
        }
        const float scale = (float)(65536 - L);
        uint32_t c[8];
#pragma unroll
        for (int q = 0; q < 8; ++q)     // rounded through 64 bits, as plane_cdf_u16
            c[q] = (e0 + q < L) ? ((uint32_t)(__float2ll_rn(__fmul_rn(acc[q], scale)) + e0 + q) & 0xFFFFu) : 0u;
#pragma unroll
        for (int q = 0; q < 8; q += 2) w[q / 2] = c[q] | (c[q + 1] << 16);
    }
    *reinterpret_cast<uint4 *>(rows + 8 * v) = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace
}  // namespace l3c

using namespace l3c;

extern "C" int l3c_batch_intervals(const l3c_code_src_t *src_dev, const int64_t *sym_off_dev, int n_streams,
                                   int64_t n_total, uint32_t *intervals_dev, int32_t *bad_dev, void *stream) {
    L3C_REQUIRE(n_streams >= 0 && n_total >= 0, "l3c_batch_intervals: n_streams=%d n_total=%lld", n_streams,
                (long long)n_total);
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(src_dev && sym_off_dev && bad_dev && (intervals_dev || n_total == 0),
                "l3c_batch_intervals: null pointer");
    const int64_t blocks = ceil_div64(n_total, BATCH_THREADS);
    L3C_REQUIRE(blocks <= INT_MAX, "l3c_batch_intervals: %lld symbols", (long long)n_total);
    cudaStream_t st = (cudaStream_t)stream;
    L3C_CUDA(cudaMemsetAsync(bad_dev, 0xFF, sizeof(int32_t) * (size_t)n_streams, st));
    if (n_total == 0) return L3C_OK;
    batch_intervals_kernel<<<(unsigned)blocks, BATCH_THREADS, 0, st>>>(src_dev, sym_off_dev, n_streams, n_total,
                                                                       intervals_dev,
                                                                       reinterpret_cast<uint32_t *>(bad_dev));
    L3C_LAUNCH_CHECK("batch_intervals_kernel");
    return L3C_OK;
}

extern "C" int l3c_batch_rows(const l3c_code_src_t *src_dev, const int64_t *row_off_dev, int n_streams,
                              int64_t n_entries, uint32_t first, uint16_t *rows_dev, void *stream) {
    L3C_REQUIRE(n_streams >= 0 && n_entries >= 0 && n_entries % 8 == 0,
                "l3c_batch_rows: n_streams=%d n_entries=%lld (a multiple of 8)", n_streams, (long long)n_entries);
    if (n_streams == 0 || n_entries == 0) return L3C_OK;
    L3C_REQUIRE(src_dev && row_off_dev && rows_dev, "l3c_batch_rows: null pointer");
    L3C_REQUIRE((reinterpret_cast<uintptr_t>(rows_dev) & 15u) == 0, "l3c_batch_rows: rows_dev must be 16-byte aligned");
    const int64_t blocks = ceil_div64(n_entries / 8, BATCH_THREADS);
    L3C_REQUIRE(blocks <= INT_MAX, "l3c_batch_rows: %lld entries", (long long)n_entries);
    batch_rows_kernel<<<(unsigned)blocks, BATCH_THREADS, 0, (cudaStream_t)stream>>>(src_dev, row_off_dev, n_streams,
                                                                                    n_entries / 8, first, rows_dev);
    L3C_LAUNCH_CHECK("batch_rows_kernel");
    return L3C_OK;
}
