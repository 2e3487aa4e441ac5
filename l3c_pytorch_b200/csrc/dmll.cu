// dmll.cu -- discretised-logistic-mixture head for sm_90a: parameter unpacking, 16-bit CDF
// quantisation, per-symbol coding intervals (encode), CDF rows (decode) and the NLL.
//
// Reference behaviour restated (files under /root/reference/src):
//   parameter layout / clamp / softmax / RGB mean coupling
//       criterion/logistic_mixture.py:134-141, 209-275
//   CDF formula and uint16 renormalisation (sequential k-sum, fp32)
//       torchac/torchac_backend/torchac_kernel.cu:16-76  (PyTorch twin: torchac/torchac.py:174-213)
//   NLL  criterion/logistic_mixture.py:146-207, 334-345
//   uniform prior row  bitcoding/bitcoding.py:297-323
//
// H100 design: the reference materialises a (H*W) x (L+1) table per channel in managed memory and
// walks it on the CPU.  Here the ENCODER never builds a table -- it evaluates the CDF only at the
// two edges of each coded symbol (20 sigmoids instead of 2570 per RGB sub-pixel) -- and the
// DECODER builds compact rows (L entries, no dead last entry) in HBM, chunk by chunk, on SMs that
// the latency-bound range decoder leaves idle.
//
// Encoder and decoder MUST see identical integers: both go through channel_params() and
// mixture_cdf_u16() below, which are written with explicit round-to-nearest intrinsics so that the
// compiler cannot contract or re-associate them differently in the two kernels.
#include "common.cuh"
#include "dmll_math.cuh"

namespace l3c {

// LOG_SCALES_MIN, sigmoid_rn, sigmoid_from_log2, ChanParams, channel_params(), mixture_cdf_u16(): dmll_math.cuh

// ---------------------------------------------------------------------------------------------
// encode side: per-symbol intervals
// ---------------------------------------------------------------------------------------------
constexpr int IV_PIX = 64;   // pixels (= threads) per CTA

// BAND: the pixels are the tile-aligned rectangle `g` (RectGeom, dmll_math.cuh) of a banded encode or a region update,
// HW = g.h * g.W; `l` is the window plane the rectangle sits in, the symbols are read from the symbol window and the
// intervals written in tile order.
// IMG (with BAND): every image n has its own rectangle, geo[n] = (oy, ox, y0, x0, h, w, ...) (RECTS_GEO ints per
// image), cut into its own tile grid; HW is then the stride of the stream-order planes (>= h * w) and g.oy, g.ox, g.y0,
// g.x0, g.h, g.W are unused (l3c_dmll_intervals_rects).
constexpr int RECTS_GEO = 10;
template <int K, bool BAND = false, bool IMG = false>
__global__ void __launch_bounds__(IV_PIX)
dmll_intervals_kernel(const float *__restrict__ l, const uint8_t *__restrict__ sym,
                      const float *__restrict__ targets, int HW, int C, int L, int rgb,
                      uint32_t *__restrict__ intervals, const RectGeom g_arg = RectGeom(),
                      const int *__restrict__ geo = nullptr) {
    extern __shared__ float sm[];
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int pitch = Kp + 1;                       // odd pitch: conflict-free column walks
    const int n = blockIdx.y;
    const int p0 = blockIdx.x * IV_PIX;
    RectGeom g = g_arg;
    int npix = HW;
    if constexpr (IMG) {
        const int *gn = geo + (size_t)n * RECTS_GEO;
        g.oy = gn[0], g.ox = gn[1], g.y0 = gn[2], g.x0 = gn[3], g.h = gn[4], g.W = gn[5];
        npix = g.h * g.W;
    }
    const int np = min(IV_PIX, npix - p0);
    if (IMG && np <= 0) return;                        // past this image's rectangle (uniform per CTA)
    if constexpr (BAND) {
        for (int i = threadIdx.x; i < np * Kp; i += IV_PIX) {
            const int j = i / Kp, pb = p0 + j, py = pb / g.W;
            const int64_t px = (int64_t)n * g.l_hw + (int64_t)(g.oy + py) * g.Wl + g.ox + (pb - py * g.W);
            sm[j * pitch + (i - j * Kp)] = l[px * Kp + (i - j * Kp)];
        }
    } else {
        const float *src = l + ((size_t)n * HW + p0) * Kp;
        for (int i = threadIdx.x; i < np * Kp; i += IV_PIX) sm[(i / Kp) * pitch + (i % Kp)] = src[i];
    }
    __syncthreads();
    if ((int)threadIdx.x >= np) return;
    const int p = p0 + threadIdx.x;
    const float *lp = sm + threadIdx.x * pitch;
    const float scale = (float)(65536 - L);         // 2^16 - (Lp - 1)
    float xr = 0.f, xg = 0.f;
    for (int c = 0; c < C; ++c) {
        ChanParams<K> cp;
        channel_params<K>(lp, 1, C, c, rgb != 0, xr, xg, cp);
        int64_t si, oi;
        if constexpr (BAND) {
            const int py = p / g.W, px = p - py * g.W;
            si = ((int64_t)n * C + c) * g.sym_hw + sym_row(g, py) + px;
            oi = ((int64_t)n * C + c) * HW + raster_to_tile_order(py, px, g.h, g.W, g.th, g.tw);
        } else {
            si = oi = ((size_t)n * C + c) * HW + p;
        }
        const int s = sym[si];
        const uint32_t lo = mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(targets + s), scale, s);
        const uint32_t hi = (s == L - 1)
                                ? 0x10000u
                                : mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(targets + s + 1),
                                                     scale, s + 1);
        intervals[oi] = lo | ((hi - 1u) << 16);
        if (c == 0) xr = (float)s;
        if (c == 1) xg = (float)s;
    }
}

// ---------------------------------------------------------------------------------------------
// decode side: CDF rows of one channel
// ---------------------------------------------------------------------------------------------
constexpr int TB_PIX = 256;      // pixels per CTA = threads: every warp takes part in the per-pixel parameter phase
                                 // (with 64 pixels per CTA, 6 of 8 warps idled through it and it dominated the kernel)
constexpr int TB_THREADS = 256;

// tile_order_to_raster, raster_to_tile_order (the tiled stream order): dmll_math.cuh

// rows (and the symbols of the already decoded channels, `sym`) are indexed in STREAM order: raster order, or
// tile order when th > 0; the parameters `l` are always read at the raster pixel.  WIN: the H x W symbol plane is
// the rectangle at (oy, ox) of a wider parameter plane of l_hw pixels per image and width Wl (a decoder window,
// l3c_dmll_build_table_window); otherwise `l` covers exactly the H x W plane and the last four arguments are unused.
// IMG (with WIN): every image n has its own rectangle, geo[n] = (oy, ox, H_n, W_n), cut into its own tile grid;
// HW is then the stride of the stream-order planes (>= H_n * W_n) and H, W, oy, ox are unused
// (l3c_dmll_build_table_windows).
template <int K, bool WIN, bool IMG = false>
__global__ void __launch_bounds__(TB_THREADS)
dmll_table_kernel(const float *__restrict__ l, const uint8_t *__restrict__ sym,
                  const float *__restrict__ targets, int HW, int C, int L, int rgb, int c_first,
                  int pix0, int npix, uint16_t *__restrict__ table, int pitch, int H, int W, int th, int tw,
                  int64_t l_hw, int Wl, int oy, int ox, const int4 *__restrict__ geo) {
    __shared__ float s_pi[TB_PIX][K];
    __shared__ float s_mu[TB_PIX][K];
    __shared__ float s_is[TB_PIX][K];
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int c = c_first + blockIdx.z;
    if (IMG) {
        const int4 g = geo[n];
        oy = g.x, ox = g.y, H = g.z, W = g.w;
        npix = H * W;
    }
    const int q0 = blockIdx.x * TB_PIX;                // offset inside [pix0, pix0+npix)
    const int np = min(TB_PIX, npix - q0);
    if (IMG && np <= 0) return;                        // past this image's rectangle (uniform per CTA)
    if ((int)threadIdx.x < np) {
        const int p = pix0 + q0 + threadIdx.x;                                     // stream-order index
        const int pr = th > 0 ? tile_order_to_raster(p, H, W, th, tw) : p;         // raster pixel
        const float *lp;
        if (WIN) {
            const int py = pr / W, px = pr - py * W;
            lp = l + ((size_t)n * l_hw + (size_t)(oy + py) * Wl + ox + px) * Kp;
        } else {
            lp = l + ((size_t)n * HW + pr) * Kp;
        }
        float xr = 0.f, xg = 0.f;
        if (rgb && c >= 1) xr = (float)sym[((size_t)n * C + 0) * HW + p];
        if (rgb && c >= 2) xg = (float)sym[((size_t)n * C + 1) * HW + p];
        ChanParams<K> cp;
        channel_params<K>(lp, 1, C, c, rgb != 0, xr, xg, cp);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            s_pi[threadIdx.x][k] = cp.pi[k];
            s_mu[threadIdx.x][k] = cp.mu[k];
            s_is[threadIdx.x][k] = cp.inv_s[k];
        }
    }
    __syncthreads();
    // One WARP per row, lanes across its entries (e = 32 j + lane): the row's 3 x K parameters are read from
    // shared memory once and stay in registers for all its entries.  (The first version spread a row over all
    // 8 warps: 30 broadcast LDS per warp and row = 240 LDS per row, and the kernel was bound by the shared-memory
    // pipe, not by its MUFU work.)
    const float scale = (float)(65536 - L);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int groups = pitch >> 5;                     // 32-entry groups per row: 1 (L <= 32) or 8
    float tg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int e = 32 * j + lane;
        tg[j] = (j < groups && e < L) ? __ldg(targets + e) : 0.f;
    }
    for (int r = warp; r < np; r += TB_THREADS / 32) {
        float pi[K], mu[K], is[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            pi[k] = s_pi[r][k];
            mu[k] = s_mu[r][k];
            is[k] = s_is[r][k];
        }
        // lane k < K also holds term k on its own: group-wide saturation tests cost one term per lane
        const float mu_l = s_mu[r][lane < K ? lane : 0], is_l = s_is[r][lane < K ? lane : 0];
        uint16_t *row = table + (((size_t)n * C + c) * HW + pix0 + q0 + r) * pitch;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j >= groups) break;
            const int e = 32 * j + lane;
            uint32_t v = 0u;
            bool done = false;
            if (32 * j + 31 < L) {                  // a whole group of valid entries
                // u = (t - mu) * is is non-increasing in t (fp subtraction and multiplication by a negative
                // constant are monotone): ALL 32 entries of the group have term k saturated low iff the first
                // one has, saturated high iff the last one has.  If every term is one or the other, the 32 CDF
                // values are the same sum of pi's (+ e): ~35 instead of ~75 instructions for the group, and
                // exactly what mixture_saturated() / mixture_cdf_u16() give lane by lane.
                const float t_first = __shfl_sync(0xFFFFFFFFu, tg[j], 0), t_last = __shfl_sync(0xFFFFFFFFu, tg[j], 31);
                const float u_first = __fmul_rn(__fsub_rn(t_first, mu_l), is_l);
                const float u_last = __fmul_rn(__fsub_rn(t_last, mu_l), is_l);
                const uint32_t lo_mask = __ballot_sync(0xFFFFFFFFu, lane < K && u_first <= SAT_LO);
                const uint32_t hi_mask = __ballot_sync(0xFFFFFFFFu, lane < K && u_last >= SAT_HI);
                if ((lo_mask | hi_mask) == (1u << K) - 1u) {
                    float acc = 0.f;
#pragma unroll
                    for (int k = 0; k < K; ++k) acc = ((lo_mask >> k) & 1u) ? __fadd_rn(acc, pi[k]) : acc;
                    v = (uint32_t)(__float2int_rn(__fmul_rn(acc, scale)) + e) & 0xFFFFu;
                    done = true;
                }
            }
            if (!done) {
                // 32 neighbouring entries of one row: where all of their terms are saturated an entry is a sum of
                // pi's -- no MUFU work for the whole warp (dmll_math.cuh)
                const bool sat = mixture_saturated<K>(pi, mu, is, tg[j], scale, e, v);
                if (!__all_sync(0xFFFFFFFFu, sat || e >= L)) v = mixture_cdf_u16<K>(pi, mu, is, tg[j], scale, e);
            }
            row[e] = (e < L) ? (uint16_t)v : (uint16_t)0;
        }
    }
}

// Coarse rows of RGB channel c (L = 256, raster stream order): per sub-pixel the record of dmll_math.cuh
// (COARSE_REC_U16) -- channel_params() exactly as dmll_table_kernel computes them, and the entries cdf[8 i].  One
// warp per record: lane l writes parameter word l and evaluates coarse entry l, 32 instead of 256 entries.
// WIN (l3c_dmll_build_coarse_windows): every image n has its own rectangle geo[n] = (oy, ox, H_n, W_n) of a decoder
// window's output, l_hw pixels per image and Wl wide; its records and the decoded symbols are in the raster order of
// the H_n x W_n rectangle, in planes of HW (>= H_n * W_n) elements, and pix0 is 0.
template <bool WIN = false>
__global__ void __launch_bounds__(TB_THREADS)
dmll_coarse_kernel(const float *__restrict__ l, const uint8_t *__restrict__ sym, const float *__restrict__ targets,
                   int HW, int c, int pix0, int npix, uint16_t *__restrict__ rec, const int4 *__restrict__ geo = nullptr,
                   int64_t l_hw = 0, int Wl = 0) {
    constexpr int K = 10, C = 3, Kp = 4 * C * K;
    __shared__ float s_par[TB_PIX][COARSE_PARAM_WORDS + 1];          // odd pitch: conflict-free column writes
    const int n = blockIdx.y;
    int oy = 0, ox = 0, w = 1;
    if constexpr (WIN) {
        const int4 g = geo[n];
        oy = g.x, ox = g.y, w = g.w;
        npix = g.z * g.w;
    }
    const int q0 = blockIdx.x * TB_PIX;
    const int np = min(TB_PIX, npix - q0);
    if (WIN && np <= 0) return;                        // past this image's rectangle (uniform per CTA)
    if ((int)threadIdx.x < np) {
        const int p = pix0 + q0 + threadIdx.x;
        const float *lp;
        if constexpr (WIN) {
            const int py = p / w, px = p - py * w;
            lp = l + ((size_t)n * l_hw + (size_t)(oy + py) * Wl + ox + px) * Kp;
        } else {
            lp = l + ((size_t)n * HW + p) * Kp;
        }
        float xr = 0.f, xg = 0.f;
        if (c >= 1) xr = (float)sym[((size_t)n * C + 0) * HW + p];
        if (c >= 2) xg = (float)sym[((size_t)n * C + 1) * HW + p];
        ChanParams<K> cp;
        channel_params<K>(lp, 1, C, c, true, xr, xg, cp);
        float *o = s_par[threadIdx.x];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            o[k] = cp.pi[k];
            o[K + k] = cp.mu[k];
            o[2 * K + k] = cp.inv_s[k];
        }
        o[3 * K] = o[3 * K + 1] = 0.f;
    }
    __syncthreads();
    const float scale = (float)(65536 - 256);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float tg = __ldg(targets + COARSE_STEP * lane);
    for (int r = warp; r < np; r += TB_THREADS / 32) {
        float pi[K], mu[K], is[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            pi[k] = s_par[r][k];
            mu[k] = s_par[r][K + k];
            is[k] = s_par[r][2 * K + k];
        }
        const uint32_t v = mixture_cdf_u16_warp<K>(pi, mu, is, tg, scale, COARSE_STEP * lane, true);
        uint16_t *out = rec + (((size_t)n * C + c) * HW + pix0 + q0 + r) * COARSE_REC_U16;
        reinterpret_cast<float *>(out)[lane] = s_par[r][lane];
        out[2 * COARSE_PARAM_WORDS + lane] = (uint16_t)v;
    }
}

// ---------------------------------------------------------------------------------------------
// reference-shaped per-channel parameters (CDFOut of logistic_mixture.py:61-65,134-141):
// softmax(pi), mu (with RGB coupling), clamped log sigma as [N][K][HW] planes
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void dmll_channel_params_kernel(const float *__restrict__ l, const float *__restrict__ x_dec,
                                           int HW, int C, int rgb, int c, float *__restrict__ pi_out,
                                           float *__restrict__ mu_out, float *__restrict__ ls_out) {
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float *lp = l + ((size_t)n * HW + p) * Kp;
    float xr = 0.f, xg = 0.f;
    if (rgb && c >= 1) xr = x_dec[((size_t)n * C + 0) * HW + p];
    if (rgb && c >= 2) xg = x_dec[((size_t)n * C + 1) * HW + p];
    ChanParams<K> cp;
    channel_params<K>(lp, 1, C, c, rgb != 0, xr, xg, cp);
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const size_t o = ((size_t)n * K + k) * HW + p;
        pi_out[o] = cp.pi[k];
        mu_out[o] = cp.mu[k];
        ls_out[o] = fmaxf(lp[2 * C * K + c * K + k], LOG_SCALES_MIN);
    }
}

// ---------------------------------------------------------------------------------------------
// NLL (theoretical bit cost)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float softplus_f(float x) {   // torch.nn.functional.softplus, threshold 20
    return (x > 20.f) ? x : log1pf(expf(x));
}

constexpr int NLL_THREADS = 128;

// Pixels of image n the NLL visits: all H*W of the plane, or (RAGGED) the h_n x w_n of its extent, which must lie
// inside the plane -- an extent that does not covers no pixel here and makes nll_finish_kernel report NaN.
__device__ __forceinline__ int nll_pixels(const int *__restrict__ extents, int n, int H, int W, int &wn) {
    if (!extents) {
        wn = W;
        return H * W;
    }
    const int hn = extents[2 * n];
    wn = extents[2 * n + 1];
    return (hn >= 1 && hn <= H && wn >= 1 && wn <= W) ? hn * wn : 0;
}

// One CTA sums NLL_THREADS consecutive pixels of one image.  Pixel q of image n is taken in raster order of the
// pixels it visits (nll_pixels): with RAGGED the plane is a padded H x W and q lies at row q / w_n, column q % w_n
// of it, so image n is cut into the same CTAs, partials and per-pixel math as a launch on that image alone.
template <int K, bool RAGGED>
__global__ void __launch_bounds__(NLL_THREADS)
dmll_nll_kernel(const float *__restrict__ l, const uint8_t *__restrict__ sym,
                const float *__restrict__ values, int H, int W, int C, int L, int rgb, float x_min,
                float x_max, const int *__restrict__ extents /* [N][2], RAGGED only */,
                double *__restrict__ partial /* [N][gridDim.x] */,
                float *__restrict__ nll_map /* [N][C][HW] or null */) {
    // first: the fp64 division is a call, and the ragged pixel mapping held across it spilled to local memory
    const float half_bin = (float)(((double)x_max - (double)x_min) / (double)(L - 1) / 2.0);
    const int HW = H * W;
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int q = blockIdx.x * NLL_THREADS + threadIdx.x;
    int wn;
    const int npix = nll_pixels(RAGGED ? extents : nullptr, n, H, W, wn);
    if (RAGGED && (int)blockIdx.x * NLL_THREADS >= npix) return;       // the whole CTA: beyond this image
    const int p = RAGGED ? q + (q / wn) * (W - wn) : q;                // row q / w_n, column q % w_n
    double mine = 0.0;
    if (q < npix) {
        const float *lp = l + ((size_t)n * HW + p) * Kp;
        float xr = 0.f, xg = 0.f;
        for (int c = 0; c < C; ++c) {
            const float x = __ldg(values + sym[((size_t)n * C + c) * HW + p]);
            const float *logit = lp + 0 * C * K + c * K;
            const float *mean = lp + 1 * C * K + c * K;
            const float *logs = lp + 2 * C * K + c * K;
            float lmax = logit[0];
#pragma unroll
            for (int k = 1; k < K; ++k) lmax = fmaxf(lmax, logit[k]);
            float lsum = 0.f;
#pragma unroll
            for (int k = 0; k < K; ++k) lsum += expf(logit[k] - lmax);
            const float lse_pi = lmax + logf(lsum);
            float w[K];
            float wmax = -INFINITY;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                float mu = mean[k];
                if (rgb && c == 1) mu += sigmoid_rn(lp[3 * C * K + 0 * K + k]) * xr;
                if (rgb && c == 2)
                    mu += sigmoid_rn(lp[3 * C * K + 1 * K + k]) * xr +
                          sigmoid_rn(lp[3 * C * K + 2 * K + k]) * xg;
                const float inv = expf(-fmaxf(logs[k], LOG_SCALES_MIN));
                const float cx = x - mu;
                const float plus_in = inv * (cx + half_bin);
                const float min_in = inv * (cx - half_bin);
                const float delta = sigmoid_rn(plus_in) - sigmoid_rn(min_in);
                float lp_k = logf(fmaxf(delta, 1e-12f));
                if (x > x_max - 0.001f) lp_k = -softplus_f(min_in);
                if (x < x_min + 0.001f) lp_k = plus_in - softplus_f(plus_in);
                w[k] = lp_k + (logit[k] - lse_pi);
                wmax = fmaxf(wmax, w[k]);
            }
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < K; ++k) s += expf(w[k] - wmax);
            const float nats = -(wmax + logf(s));
            if (nll_map) nll_map[((size_t)n * C + c) * HW + p] = nats;
            mine += (double)nats;
            if (c == 0) xr = x;
            if (c == 1) xg = x;
        }
    }
    // deterministic block reduction (fixed tree), one partial per CTA
    __shared__ double red[NLL_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < NLL_THREADS / 32; ++i) t += red[i];
        partial[(size_t)n * gridDim.x + blockIdx.x] = t;
    }
}

__global__ void nll_finish_kernel(const double *__restrict__ partial, int per_image, int H, int W,
                                  const int *__restrict__ extents, double *__restrict__ out) {
    // one warp per image, fixed summation order; a ragged image sums only the partials of its own CTAs
    const int n = blockIdx.x;
    int count = per_image, wn;
    if (extents) {
        const int npix = nll_pixels(extents, n, H, W, wn);
        if (npix == 0) {
            if (threadIdx.x == 0) out[n] = __longlong_as_double(0x7FF8000000000000LL);
            return;
        }
        count = (npix + NLL_THREADS - 1) / NLL_THREADS;
    }
    double t = 0.0;
    for (int i = threadIdx.x; i < count; i += 32) t += partial[(size_t)n * per_image + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xFFFFFFFFu, t, o);
    if (threadIdx.x == 0) out[n] = t;
}

// ---------------------------------------------------------------------------------------------
// training (DESIGN §4.9): the DMLL loss of train.dmll_nll and its gradient, and the soft quantiser, on the NCHW fp32
// tensors nn.Conv2d produces.  l [N][Kp][HW] (channel p*C*K + c*K + k), x [N][C][HW] float targets.  One thread per
// pixel walks the Kp planes, so every load and store of a warp is one coalesced line per plane.  The backward
// recomputes everything from l and x: nothing but the two inputs is kept between the passes.
// ---------------------------------------------------------------------------------------------
// One mixture component as train.dmll_nll evaluates it in fp32 (logistic_mixture.py:146-207): the sigmoid arguments
// u+ / u- at the two bin edges, their sigmoids, delta = s+ - s- and the component's log-probability lp (middle branch
// log(max(delta, 1e-12)); x above x_upper: -softplus(u-); x below x_lower: u+ - softplus(u+), applied last).
struct TrainTerm {
    float inv, up, um, sp, sm, delta, lp;
};

__device__ __forceinline__ TrainTerm train_term(float x, float mu, float ls_raw, float half_bin, bool hi, bool lo) {
    TrainTerm t;
    t.inv = expf(-fmaxf(ls_raw, LOG_SCALES_MIN));
    const float cx = __fsub_rn(x, mu);
    t.up = __fmul_rn(t.inv, __fadd_rn(cx, half_bin));
    t.um = __fmul_rn(t.inv, __fsub_rn(cx, half_bin));
    t.sp = sigmoid_rn(t.up);
    t.sm = sigmoid_rn(t.um);
    t.delta = __fsub_rn(t.sp, t.sm);
    float lp = logf(fmaxf(t.delta, 1e-12f));
    if (hi) lp = -softplus_f(t.um);
    if (lo) lp = __fsub_rn(t.up, softplus_f(t.up));
    t.lp = lp;
    return t;
}

// The effective mean of component k of channel c: RGB channels 1 and 2 add sigmoid(coeff) times the targets of the
// channels before them, in torch's order ((mean + co_br x0) + co_bg x1).  lp: the pixel's plane 0, stride HW.
template <int K>
__device__ __forceinline__ float train_mean(const float *__restrict__ lp, int64_t HW, int C, int c, int k, bool rgb,
                                            float x0, float x1) {
    float mu = __ldg(lp + (int64_t)(1 * C * K + c * K + k) * HW);
    const float *co = lp + (int64_t)3 * C * K * HW;
    if (rgb && c == 1) mu = __fadd_rn(mu, __fmul_rn(sigmoid_rn(__ldg(co + (int64_t)(0 * K + k) * HW)), x0));
    if (rgb && c == 2) {
        mu = __fadd_rn(mu, __fmul_rn(sigmoid_rn(__ldg(co + (int64_t)(1 * K + k) * HW)), x0));
        mu = __fadd_rn(mu, __fmul_rn(sigmoid_rn(__ldg(co + (int64_t)(2 * K + k) * HW)), x1));
    }
    return mu;
}

// Channel c of one pixel: w[k] = lp_k + log_softmax(logits)_k, -> nats = -logsumexp_k w_k; also the logits'
// log-sum-exp and w's maximum and sum of exponentials, from which the backward takes the two softmaxes.
template <int K>
__device__ __forceinline__ float train_channel(const float *__restrict__ lp, int64_t HW, int C, int c, bool rgb,
                                               float xc, float x0, float x1, float half_bin, bool hi, bool lo,
                                               float (&w)[K], float &lse_pi, float &wmax, float &wsum) {
    const float *logit = lp + (int64_t)(c * K) * HW;
    const float *logs = lp + (int64_t)(2 * C * K + c * K) * HW;
    float lg[K];
#pragma unroll
    for (int k = 0; k < K; ++k) lg[k] = __ldg(logit + (int64_t)k * HW);
    float lmax = lg[0];
#pragma unroll
    for (int k = 1; k < K; ++k) lmax = fmaxf(lmax, lg[k]);
    float lsum = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) lsum += expf(lg[k] - lmax);
    lse_pi = lmax + logf(lsum);
    wmax = -INFINITY;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float mu = train_mean<K>(lp, HW, C, c, k, rgb, x0, x1);
        const TrainTerm t = train_term(xc, mu, __ldg(logs + (int64_t)k * HW), half_bin, hi, lo);
        w[k] = t.lp + (lg[k] - lse_pi);
        wmax = fmaxf(wmax, w[k]);
    }
    wsum = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) wsum += expf(w[k] - wmax);
    return -(wmax + logf(wsum));
}

// Forward: the nats of every sub-pixel summed per CTA in f64, in the fixed order of dmll_nll_kernel; the per-image
// totals then come from nll_finish_kernel.
template <int K>
__global__ void __launch_bounds__(NLL_THREADS)
dmll_train_nll_kernel(const float *__restrict__ l, const float *__restrict__ x, int HW, int C, int rgb, float half_bin,
                      float x_lower, float x_upper, double *__restrict__ partial /* [N][gridDim.x] */) {
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int p = blockIdx.x * NLL_THREADS + threadIdx.x;
    double mine = 0.0;
    if (p < HW) {
        const float *lp = l + (int64_t)n * Kp * HW + p;
        const float *xp = x + (int64_t)n * C * HW + p;
        const float x0 = rgb ? __ldg(xp) : 0.f, x1 = rgb ? __ldg(xp + HW) : 0.f;
        for (int c = 0; c < C; ++c) {
            const float xc = __ldg(xp + (int64_t)c * HW);
            float w[K], lse_pi, wmax, wsum;
            mine += (double)train_channel<K>(lp, HW, C, c, rgb != 0, xc, x0, x1, half_bin, xc > x_upper,
                                             xc < x_lower, w, lse_pi, wmax, wsum);
        }
    }
    __shared__ double red[NLL_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_down_sync(0xFFFFFFFFu, mine, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < NLL_THREADS / 32; ++i) t += red[i];
        partial[(size_t)n * gridDim.x + blockIdx.x] = t;
    }
}

// Backward of the summed nats for the upstream gradient *grad: every element of dl (all Kp planes) and of dx (non-RGB,
// optional) is written once by the thread of its pixel -- no atomics, the same bits on every run.  With r = softmax(w)
// and pi = softmax(logits): dlogit = g (pi - r); e = -g r is the gradient of lp, which reaches u+ / u- as a+ / a- on
// the branch taken (0 on the others, and 0 on the middle branch where delta < 1e-12, as torch.clamp's gradient);
// dmean = -inv (a+ + a-), dlogscale = -(u+ a+ + u- a-) where the raw log-scale is >= -7, dx = sum_k inv (a+ + a-);
// RGB: dcoeff = dmean of the channel it couples into, times the target it multiplies, times sigmoid'(coeff).
// sigmoid' is s (1 - s) and the lower branch's slope 1 - s, from the same fp32 s as delta, as torch's autograd
// forms them: where s+ - s- cancels, the rounding of 1 - s and of delta then go together as in the torch path
// (sigmoid(u) sigmoid(-u) is closer to float64 per element, but moved the encoder's gradients of a step at
// initialisation by up to 2 % away from the reference's, as many sub-pixels sit in that regime there).
template <int K>
__global__ void __launch_bounds__(NLL_THREADS)
dmll_train_grad_kernel(const float *__restrict__ l, const float *__restrict__ x, int HW, int C, int rgb,
                       float half_bin, float x_lower, float x_upper, const float *__restrict__ grad,
                       float *__restrict__ dl, float *__restrict__ dx) {
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int p = blockIdx.x * NLL_THREADS + threadIdx.x;
    if (p >= HW) return;
    const float g = __ldg(grad);
    const float *lp = l + (int64_t)n * Kp * HW + p;
    float *dlp = dl + (int64_t)n * Kp * HW + p;
    const float *xp = x + (int64_t)n * C * HW + p;
    const float x0 = rgb ? __ldg(xp) : 0.f, x1 = rgb ? __ldg(xp + HW) : 0.f;
    for (int c = 0; c < C; ++c) {
        const float xc = __ldg(xp + (int64_t)c * HW);
        const bool hi = xc > x_upper, lo = xc < x_lower;
        float w[K], lse_pi, wmax, wsum;
        train_channel<K>(lp, HW, C, c, rgb != 0, xc, x0, x1, half_bin, hi, lo, w, lse_pi, wmax, wsum);
        float dxc = 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int64_t i_logit = c * K + k, i_mean = C * K + c * K + k, i_ls = 2 * C * K + c * K + k;
            const float r = expf(w[k] - wmax) / wsum;
            const float pi = expf(__ldg(lp + i_logit * HW) - lse_pi);
            dlp[i_logit * HW] = g * (pi - r);
            const float e = -g * r;
            const float ls_raw = __ldg(lp + i_ls * HW);
            const TrainTerm t = train_term(xc, train_mean<K>(lp, HW, C, c, k, rgb != 0, x0, x1), ls_raw, half_bin,
                                           hi, lo);
            float ap = 0.f, am = 0.f;
            if (lo) {
                ap = (t.up > 20.f) ? 0.f : e * (1.f - t.sp);                 // d(u - softplus u) = 1 - sigmoid(u)
            } else if (hi) {
                am = -e * ((t.um > 20.f) ? 1.f : t.sm);                      // d softplus(u) = sigmoid(u)
            } else if (t.delta >= 1e-12f) {
                const float q = e / t.delta;
                ap = q * (t.sp * (1.f - t.sp));                              // sigmoid' = s (1 - s), as torch
                am = -q * (t.sm * (1.f - t.sm));
            }
            const float s = ap + am;
            const float dmean = -t.inv * s;
            dlp[i_mean * HW] = dmean;
            dlp[i_ls * HW] = (ls_raw >= LOG_SCALES_MIN) ? -(t.up * ap + t.um * am) : 0.f;
            dxc += t.inv * s;
            if (rgb && c > 0) {
                // channel 1 couples through coefficient plane 0 (x0); channel 2 through planes 1 (x0) and 2 (x1)
                const int64_t j0 = 3 * C * K + (c == 1 ? 0 : 1) * K + k;
                const float s0 = sigmoid_rn(__ldg(lp + j0 * HW));
                dlp[j0 * HW] = dmean * x0 * (s0 * (1.f - s0));
                if (c == 2) {
                    const int64_t j1 = 3 * C * K + 2 * K + k;
                    const float s1 = sigmoid_rn(__ldg(lp + j1 * HW));
                    dlp[j1 * HW] = dmean * x1 * (s1 * (1.f - s1));
                }
            }
        }
        if (!rgb && dx) dx[((int64_t)n * C + c) * HW + p] = dxc;
    }
}

// Soft quantiser (quantizer.py:62-90).  Forward: sym = the first argmin of (q - c_l)^2 (strict <, as torch.min and
// quantize_head_kernel take it), value = levels[sym].  Backward: d value_soft / dq for value_soft = sum_l c_l phi_l,
// phi = softmax_l(-sigma (q - c_l)^2), is 2 sigma Var_phi(c), evaluated centred (sum_l phi_l (c_l - cbar)^2).
constexpr int SQ_THREADS = 256;

__global__ void __launch_bounds__(SQ_THREADS)
soft_quantize_kernel(const float *__restrict__ q, int64_t n, const float *__restrict__ levels, int L, float sigma,
                     int64_t *__restrict__ sym, float *__restrict__ value, const float *__restrict__ grad,
                     float *__restrict__ dq) {
    extern __shared__ float slev[];
    for (int i = threadIdx.x; i < L; i += SQ_THREADS) slev[i] = levels[i];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * SQ_THREADS + threadIdx.x;
    if (i >= n) return;
    const float v = __ldg(q + i);
    int best = 0;
    float bd = __fmul_rn(__fsub_rn(v, slev[0]), __fsub_rn(v, slev[0]));
    for (int j = 1; j < L; ++j) {
        const float d = __fmul_rn(__fsub_rn(v, slev[j]), __fsub_rn(v, slev[j]));
        if (d < bd) {
            bd = d;
            best = j;
        }
    }
    if (!grad) {
        sym[i] = best;
        value[i] = slev[best];
        return;
    }
    // the largest logit -sigma d is the nearest level's (sigma > 0)
    const float m = -sigma * bd;
    float s = 0.f, sc = 0.f;
    for (int j = 0; j < L; ++j) {
        const float d = __fmul_rn(__fsub_rn(v, slev[j]), __fsub_rn(v, slev[j]));
        const float ph = expf(-sigma * d - m);
        s += ph;
        sc += ph * slev[j];
    }
    const float cbar = sc / s;
    float var = 0.f;
    for (int j = 0; j < L; ++j) {
        const float d = __fmul_rn(__fsub_rn(v, slev[j]), __fsub_rn(v, slev[j]));
        const float dc = slev[j] - cbar;
        var += expf(-sigma * d - m) * dc * dc;
    }
    dq[i] = __ldg(grad + i) * (2.f * sigma * (var / s));
}

// ---------------------------------------------------------------------------------------------
// sampling from the mixture (logistic_mixture.py:277-323): Gumbel-max choice of the component, inverse-CDF
// sample of its logistic, RGB means coupled through the coefficients of the CHOSEN components.  The uniform
// random numbers are inputs (u_sel [N][C][K][HW], u_x [N][C][HW], both in [1e-5, 1 - 1e-5] as in the
// reference), so the kernel is a deterministic function that a test can restate.
// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void dmll_sample_kernel(const float *__restrict__ l, const float *__restrict__ u_sel,
                                   const float *__restrict__ u_x, int HW, int C, int rgb,
                                   float *__restrict__ x_out /* [N][C][HW] */) {
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int n = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float *lp = l + ((size_t)n * HW + p) * Kp;
    float x[3] = {0.f, 0.f, 0.f};
    int sel[3] = {0, 0, 0};
    for (int c = 0; c < C; ++c) {
        int best = 0;
        float best_v = -INFINITY;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const float u = u_sel[(((size_t)n * C + c) * K + k) * HW + p];
            const float v = lp[c * K + k] - logf(-logf(u));            // Gumbel-max
            if (v > best_v) { best_v = v; best = k; }
        }
        const float mean = lp[C * K + c * K + best];
        const float ls = fmaxf(lp[2 * C * K + c * K + best], LOG_SCALES_MIN);
        const float u = u_x[((size_t)n * C + c) * HW + p];
        const float v = mean + expf(ls) * (logf(u) - logf(1.f - u));   // inverse transform sampling
        if (rgb) {
            sel[c] = best;
            x[c] = v;
        } else {
            x_out[((size_t)n * C + c) * HW + p] = v;
        }
    }
    if (rgb) {
        // coefficients of the G and B components that were chosen (logistic_mixture.py:305-320)
        const float *co = lp + 3 * C * K;
        const float c_gr = sigmoid_rn(co[0 * K + sel[1]]);
        const float c_br = sigmoid_rn(co[1 * K + sel[2]]);
        const float c_bg = sigmoid_rn(co[2 * K + sel[2]]);
        const float x0 = fminf(fmaxf(x[0], 0.f), 255.f);
        const float x1 = fminf(fmaxf(x[1] + c_gr * x0, 0.f), 255.f);
        const float x2 = fminf(fmaxf(x[2] + c_br * x0 + c_bg * x1, 0.f), 255.f);
        x_out[((size_t)n * C + 0) * HW + p] = x0;
        x_out[((size_t)n * C + 1) * HW + p] = x1;
        x_out[((size_t)n * C + 2) * HW + p] = x2;
    }
}

static int check_common(const char *fn, int N, int HW, int C, int K, int L, int rgb) {
    L3C_REQUIRE(N >= 1 && HW >= 1, "%s: N=%d HW=%d", fn, N, HW);
    L3C_REQUIRE(K == 10, "%s: only K=10 mixtures are built (configs/ms/cr.cf:35), got K=%d", fn, K);
    L3C_REQUIRE(C >= 1 && C <= 16, "%s: C=%d", fn, C);
    L3C_REQUIRE(!rgb || C == 3, "%s: RGB coupling needs C==3 (logistic_mixture.py:236), got %d", fn, C);
    L3C_REQUIRE(L >= 2 && L <= 256, "%s: L=%d", fn, L);
    L3C_REQUIRE(N <= 65535, "%s: N=%d exceeds grid.y", fn, N);
    return L3C_OK;
}

}  // namespace l3c

extern "C" int l3c_uniform_cdf_row(int L, uint16_t *row_host) {
    using namespace l3c;
    L3C_REQUIRE(L >= 1 && L <= 256 && row_host, "l3c_uniform_cdf_row: L=%d", L);
    // bitcoding.py:297-323: fp32 ones(L)/L, fp32 cumsum, *2^16, round-half-even, int16 wrap
    const float pr = 1.0f / (float)L;
    float c = 0.f;
    row_host[0] = 0;
    for (int i = 0; i < L; ++i) {
        c += pr;
        const long v = lrintf(c * 65536.0f);
        row_host[i + 1] = (uint16_t)(v & 0xFFFF);
    }
    return L3C_OK;
}

extern "C" int l3c_dmll_intervals(const float *l_dev, const uint8_t *sym_dev,
                                  const float *targets_dev, int N, int HW, int C, int K, int L,
                                  int rgb, uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_intervals", N, HW, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && sym_dev && targets_dev && intervals_dev, "l3c_dmll_intervals: null pointer");
    const int Kp = (rgb ? 4 : 3) * C * K;
    const size_t smem = (size_t)IV_PIX * (Kp + 1) * sizeof(float);
    L3C_REQUIRE(smem <= 48 * 1024, "l3c_dmll_intervals: Kp=%d too large", Kp);
    dim3 grid(ceil_div(HW, IV_PIX), N);
    dmll_intervals_kernel<10><<<grid, IV_PIX, smem, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, HW, C, L, rgb, intervals_dev);
    L3C_LAUNCH_CHECK("dmll_intervals_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_intervals_rect(const float *l_dev, int Hl, int Wl, int oy, int ox, const uint8_t *sym_dev,
                                       int Hs, int Ws, int y0, int x0, int h, int w, int sy, int sx, int Hf, int Wf,
                                       const float *targets_dev, int N, int C, int K, int L, int rgb, int th, int tw,
                                       uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(h >= 1 && w >= 1 && (int64_t)h * w < (1ll << 31), "l3c_dmll_intervals_rect: %dx%d rectangle", h, w);
    if (int e = check_common("l3c_dmll_intervals_rect", N, h * w, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && sym_dev && targets_dev && intervals_dev, "l3c_dmll_intervals_rect: null pointer");
    L3C_REQUIRE(th >= 1 && tw >= 1, "l3c_dmll_intervals_rect: tile %dx%d", th, tw);
    L3C_REQUIRE(oy >= 0 && ox >= 0 && (int64_t)oy + h <= Hl && (int64_t)ox + w <= Wl,
                "l3c_dmll_intervals_rect: %dx%d rectangle at (%d, %d) outside the %dx%d parameter plane", h, w, oy, ox,
                Hl, Wl);
    L3C_REQUIRE(y0 >= 0 && x0 >= 0 && (int64_t)y0 + h <= Hs && (int64_t)x0 + w <= Ws,
                "l3c_dmll_intervals_rect: %dx%d rectangle at (%d, %d) outside the %dx%d symbol plane", h, w, y0, x0, Hs,
                Ws);
    L3C_REQUIRE(sy >= 0 && sx >= 0 && (int64_t)sy + Hs <= Hf && (int64_t)sx + Ws <= Wf,
                "l3c_dmll_intervals_rect: %dx%d symbol window at (%d, %d) outside the %dx%d plane", Hs, Ws, sy, sx, Hf, Wf);
    // tile-aligned in the whole plane: starts on a tile boundary, ends on one or at the plane's edge, so the
    // rectangle's tile order is that of the plane's own tiles
    const int ry = sy + y0, rx = sx + x0;
    L3C_REQUIRE(ry % th == 0 && rx % tw == 0 && ((ry + h) % th == 0 || ry + h == Hf) && ((rx + w) % tw == 0 || rx + w == Wf),
                "l3c_dmll_intervals_rect: %dx%d rectangle at (%d, %d) of a %dx%d plane is not aligned to %dx%d tiles",
                h, w, ry, rx, Hf, Wf, th, tw);
    const int Kp = (rgb ? 4 : 3) * C * K;
    const size_t smem = (size_t)IV_PIX * (Kp + 1) * sizeof(float);
    L3C_REQUIRE(smem <= 48 * 1024, "l3c_dmll_intervals_rect: Kp=%d too large", Kp);
    RectGeom g;
    g.sym_hw = (long long)Hs * Ws; g.l_hw = (long long)Hl * Wl;
    g.y0 = y0; g.h = h; g.W = w; g.Wl = Wl; g.oy = oy; g.ox = ox; g.th = th; g.tw = tw;
    g.x0 = x0; g.Ws = Ws;
    dim3 grid(ceil_div(h * w, IV_PIX), N);
    dmll_intervals_kernel<10, true><<<grid, IV_PIX, smem, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, h * w, C, L, rgb, intervals_dev, g);
    L3C_LAUNCH_CHECK("dmll_intervals_rect_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_intervals_rects(const float *l_dev, int Hl, int Wl, const uint8_t *sym_dev, int Hs, int Ws,
                                        const int *geo_host, int *geo_dev, int plane, const float *targets_dev, int N,
                                        int C, int K, int L, int rgb, int th, int tw, uint32_t *intervals_dev,
                                        void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_intervals_rects", N, plane, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && sym_dev && targets_dev && intervals_dev && geo_host && geo_dev,
                "l3c_dmll_intervals_rects: null pointer");
    L3C_REQUIRE(th >= 1 && tw >= 1 && Hl >= 1 && Wl >= 1 && Hs >= 1 && Ws >= 1,
                "l3c_dmll_intervals_rects: tile %dx%d, %dx%d parameter plane, %dx%d symbol plane", th, tw, Hl, Wl, Hs,
                Ws);
    L3C_REQUIRE(((uintptr_t)geo_dev & 3) == 0, "l3c_dmll_intervals_rects: geo_dev must be 4-byte aligned");
    int max_hw = 0;
    for (int n = 0; n < N; ++n) {
        const int *g = geo_host + (size_t)n * RECTS_GEO;
        const int oy = g[0], ox = g[1], y0 = g[2], x0 = g[3], h = g[4], w = g[5], sy = g[6], sx = g[7], Hf = g[8],
                  Wf = g[9];
        L3C_REQUIRE(h >= 1 && w >= 1 && (int64_t)h * w <= plane,
                    "l3c_dmll_intervals_rects: image %d: %dx%d rectangle, planes of %d", n, h, w, plane);
        L3C_REQUIRE(oy >= 0 && ox >= 0 && (int64_t)oy + h <= Hl && (int64_t)ox + w <= Wl,
                    "l3c_dmll_intervals_rects: image %d: %dx%d rectangle at (%d, %d) outside the %dx%d parameter plane",
                    n, h, w, oy, ox, Hl, Wl);
        L3C_REQUIRE(y0 >= 0 && x0 >= 0 && (int64_t)y0 + h <= Hs && (int64_t)x0 + w <= Ws,
                    "l3c_dmll_intervals_rects: image %d: %dx%d rectangle at (%d, %d) outside the %dx%d symbol plane", n,
                    h, w, y0, x0, Hs, Ws);
        L3C_REQUIRE(sy >= 0 && sx >= 0 && (int64_t)sy + y0 + h <= Hf && (int64_t)sx + x0 + w <= Wf,
                    "l3c_dmll_intervals_rects: image %d: symbol window at (%d, %d) puts the rectangle outside the %dx%d "
                    "plane", n, sy, sx, Hf, Wf);
        const int ry = sy + y0, rx = sx + x0;
        L3C_REQUIRE(ry % th == 0 && rx % tw == 0 && ((ry + h) % th == 0 || ry + h == Hf) &&
                        ((rx + w) % tw == 0 || rx + w == Wf),
                    "l3c_dmll_intervals_rects: image %d: %dx%d rectangle at (%d, %d) of a %dx%d plane is not aligned to "
                    "%dx%d tiles", n, h, w, ry, rx, Hf, Wf, th, tw);
        max_hw = h * w > max_hw ? h * w : max_hw;
    }
    const int Kp = (rgb ? 4 : 3) * C * K;
    const size_t smem = (size_t)IV_PIX * (Kp + 1) * sizeof(float);
    L3C_REQUIRE(smem <= 48 * 1024, "l3c_dmll_intervals_rects: Kp=%d too large", Kp);
    cudaStream_t st = (cudaStream_t)stream;
    // from pageable memory: returns once geo_host has been read, so the caller may free it
    L3C_REQUIRE(cudaMemcpyAsync(geo_dev, geo_host, (size_t)N * RECTS_GEO * sizeof(int), cudaMemcpyHostToDevice, st) ==
                    cudaSuccess, "l3c_dmll_intervals_rects: geometry upload failed");
    RectGeom g;
    g.sym_hw = (long long)Hs * Ws; g.l_hw = (long long)Hl * Wl;
    g.y0 = 0; g.h = 0; g.W = 0; g.Wl = Wl; g.oy = 0; g.ox = 0; g.th = th; g.tw = tw;
    g.x0 = 0; g.Ws = Ws;
    dim3 grid(ceil_div(max_hw, IV_PIX), N);
    dmll_intervals_kernel<10, true, true><<<grid, IV_PIX, smem, st>>>(
        l_dev, sym_dev, targets_dev, plane, C, L, rgb, intervals_dev, g, geo_dev);
    L3C_LAUNCH_CHECK("dmll_intervals_rects_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_table(const float *l_dev, const uint8_t *sym_dev,
                                    const float *targets_dev, int N, int HW, int C, int K, int L,
                                    int rgb, int c, int pix0, int npix, uint16_t *table_dev,
                                    int pitch, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_build_table", N, HW, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && targets_dev && table_dev, "l3c_dmll_build_table: null pointer");
    L3C_REQUIRE(!(rgb && c > 0) || sym_dev, "l3c_dmll_build_table: decoded symbols needed for c>0");
    L3C_REQUIRE(c < C && (c >= 0 || !rgb), "l3c_dmll_build_table: c=%d C=%d rgb=%d", c, C, rgb);
    L3C_REQUIRE((pitch == 32 && L <= 32) || (pitch == 256 && L <= 256 && L > 32),
                "l3c_dmll_build_table: pitch=%d must be 32 (L<=32) or 256, L=%d", pitch, L);
    L3C_REQUIRE(pix0 >= 0 && npix >= 0 && pix0 + npix <= HW, "l3c_dmll_build_table: pixel range");
    if (npix == 0) return L3C_OK;
    dim3 grid(ceil_div(npix, TB_PIX), N, c < 0 ? C : 1);
    dmll_table_kernel<10, false><<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, HW, C, L, rgb, c < 0 ? 0 : c, pix0, npix, table_dev, pitch, 0, 0, 0, 0, 0, 0, 0,
        0, nullptr);
    L3C_LAUNCH_CHECK("dmll_table_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_coarse(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev, int N,
                                     int HW, int K, int L, int c, int pix0, int npix, uint16_t *rec_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_build_coarse", N, HW, 3, K, L, 1)) return e;
    L3C_REQUIRE(L == 256, "l3c_dmll_build_coarse: coarse rows exist for L=256 only, got L=%d", L);
    L3C_REQUIRE(l_dev && targets_dev && rec_dev, "l3c_dmll_build_coarse: null pointer");
    L3C_REQUIRE(c >= 0 && c < 3 && (c == 0 || sym_dev), "l3c_dmll_build_coarse: c=%d (decoded symbols needed for c>0)", c);
    L3C_REQUIRE(pix0 >= 0 && npix >= 0 && pix0 + npix <= HW, "l3c_dmll_build_coarse: pixel range");
    if (npix == 0) return L3C_OK;
    dim3 grid(ceil_div(npix, TB_PIX), N);
    dmll_coarse_kernel<<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(l_dev, sym_dev, targets_dev, HW, c, pix0, npix,
                                                                      rec_dev);
    L3C_LAUNCH_CHECK("dmll_coarse_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_coarse_windows(const float *l_dev, int Hl, int Wl, const int *geo_dev, int max_hw,
                                             int plane, const uint8_t *sym_dev, const float *targets_dev, int N,
                                             int K, int L, int c, uint16_t *rec_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_build_coarse_windows", N, plane, 3, K, L, 1)) return e;
    L3C_REQUIRE(L == 256, "l3c_dmll_build_coarse_windows: coarse rows exist for L=256 only, got L=%d", L);
    L3C_REQUIRE(l_dev && targets_dev && rec_dev && geo_dev, "l3c_dmll_build_coarse_windows: null pointer");
    L3C_REQUIRE(c >= 0 && c < 3 && (c == 0 || sym_dev),
                "l3c_dmll_build_coarse_windows: c=%d (decoded symbols needed for c>0)", c);
    L3C_REQUIRE(Hl >= 1 && Wl >= 1 && max_hw >= 1 && max_hw <= plane,
                "l3c_dmll_build_coarse_windows: %dx%d parameter plane, max_hw=%d plane=%d", Hl, Wl, max_hw, plane);
    L3C_REQUIRE(((uintptr_t)geo_dev & 15) == 0, "l3c_dmll_build_coarse_windows: geo must be 16-byte aligned");
    dim3 grid(ceil_div(max_hw, TB_PIX), N);
    dmll_coarse_kernel<true><<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, plane, c, 0, 0, rec_dev, (const int4 *)geo_dev, (int64_t)Hl * Wl, Wl);
    L3C_LAUNCH_CHECK("dmll_coarse_windows_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_table_tiled(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev,
                                          int N, int H, int W, int C, int K, int L, int rgb, int c, int th, int tw,
                                          uint16_t *table_dev, int pitch, void *stream) {
    using namespace l3c;
    const int HW = H * W;
    if (int e = check_common("l3c_dmll_build_table_tiled", N, HW, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && targets_dev && table_dev, "l3c_dmll_build_table_tiled: null pointer");
    L3C_REQUIRE(!(rgb && c > 0) || sym_dev, "l3c_dmll_build_table_tiled: decoded symbols needed for c>0");
    L3C_REQUIRE(c < C && (c >= 0 || !rgb), "l3c_dmll_build_table_tiled: c=%d C=%d rgb=%d", c, C, rgb);
    L3C_REQUIRE((pitch == 32 && L <= 32) || (pitch == 256 && L <= 256 && L > 32),
                "l3c_dmll_build_table_tiled: pitch=%d must be 32 (L<=32) or 256, L=%d", pitch, L);
    L3C_REQUIRE(th >= 1 && tw >= 1 && H >= 1 && W >= 1, "l3c_dmll_build_table_tiled: tile %dx%d", th, tw);
    dim3 grid(ceil_div(HW, TB_PIX), N, c < 0 ? C : 1);
    dmll_table_kernel<10, false><<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, HW, C, L, rgb, c < 0 ? 0 : c, 0, HW, table_dev, pitch, H, W, th, tw, 0, 0, 0, 0,
        nullptr);
    L3C_LAUNCH_CHECK("dmll_table_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_table_window(const float *l_dev, int Hl, int Wl, int oy, int ox, const uint8_t *sym_dev,
                                           const float *targets_dev, int N, int H, int W, int C, int K, int L, int rgb,
                                           int c, int th, int tw, uint16_t *table_dev, int pitch, void *stream) {
    using namespace l3c;
    const int HW = H * W;
    if (int e = check_common("l3c_dmll_build_table_window", N, HW, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && targets_dev && table_dev, "l3c_dmll_build_table_window: null pointer");
    L3C_REQUIRE(!(rgb && c > 0) || sym_dev, "l3c_dmll_build_table_window: decoded symbols needed for c>0");
    L3C_REQUIRE(c < C && (c >= 0 || !rgb), "l3c_dmll_build_table_window: c=%d C=%d rgb=%d", c, C, rgb);
    L3C_REQUIRE((pitch == 32 && L <= 32) || (pitch == 256 && L <= 256 && L > 32),
                "l3c_dmll_build_table_window: pitch=%d must be 32 (L<=32) or 256, L=%d", pitch, L);
    L3C_REQUIRE(th >= 1 && tw >= 1 && H >= 1 && W >= 1, "l3c_dmll_build_table_window: tile %dx%d", th, tw);
    L3C_REQUIRE(oy >= 0 && ox >= 0 && oy + H <= Hl && ox + W <= Wl,
                "l3c_dmll_build_table_window: %dx%d rectangle at (%d, %d) outside the %dx%d parameter plane", H, W, oy,
                ox, Hl, Wl);
    dim3 grid(ceil_div(HW, TB_PIX), N, c < 0 ? C : 1);
    dmll_table_kernel<10, true><<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, HW, C, L, rgb, c < 0 ? 0 : c, 0, HW, table_dev, pitch, H, W, th, tw,
        (int64_t)Hl * Wl, Wl, oy, ox, nullptr);
    L3C_LAUNCH_CHECK("dmll_table_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_build_table_windows(const float *l_dev, int Hl, int Wl, const int *geo_dev, int max_hw,
                                            int plane, const uint8_t *sym_dev, const float *targets_dev, int N, int C,
                                            int K, int L, int rgb, int c, int th, int tw, uint16_t *table_dev,
                                            int pitch, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_build_table_windows", N, plane, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && targets_dev && table_dev && geo_dev, "l3c_dmll_build_table_windows: null pointer");
    L3C_REQUIRE(!(rgb && c > 0) || sym_dev, "l3c_dmll_build_table_windows: decoded symbols needed for c>0");
    L3C_REQUIRE(c < C && (c >= 0 || !rgb), "l3c_dmll_build_table_windows: c=%d C=%d rgb=%d", c, C, rgb);
    L3C_REQUIRE((pitch == 32 && L <= 32) || (pitch == 256 && L <= 256 && L > 32),
                "l3c_dmll_build_table_windows: pitch=%d must be 32 (L<=32) or 256, L=%d", pitch, L);
    L3C_REQUIRE(th >= 1 && tw >= 1 && Hl >= 1 && Wl >= 1 && max_hw >= 1 && max_hw <= plane,
                "l3c_dmll_build_table_windows: tile %dx%d, %dx%d parameter plane, max_hw=%d plane=%d", th, tw, Hl, Wl,
                max_hw, plane);
    L3C_REQUIRE(((uintptr_t)geo_dev & 15) == 0, "l3c_dmll_build_table_windows: geo must be 16-byte aligned");
    dim3 grid(ceil_div(max_hw, TB_PIX), N, c < 0 ? C : 1);
    dmll_table_kernel<10, true, true><<<grid, TB_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, targets_dev, plane, C, L, rgb, c < 0 ? 0 : c, 0, 0, table_dev, pitch, 0, 0, th, tw,
        (int64_t)Hl * Wl, Wl, 0, 0, (const int4 *)geo_dev);
    L3C_LAUNCH_CHECK("dmll_table_kernel");
    return L3C_OK;
}

namespace l3c {
// raster <-> tile order of `planes` planes of H x W elements of 1 or 4 bytes
template <typename T>
__global__ void reorder_tiles_kernel(const T *__restrict__ src, T *__restrict__ dst, int HW, int H, int W, int th,
                                     int tw, int to_tiles) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= HW) return;
    const size_t base = (size_t)blockIdx.y * HW;
    const int p = tile_order_to_raster((int)r, H, W, th, tw);
    if (to_tiles) dst[base + r] = src[base + p];
    else dst[base + p] = src[base + r];
}

// the h x w rectangle at origins[n] of every plane of image n (planes H x W of per_elem words or bytes)
template <typename T>
__global__ void crop_rect_kernel(const T *__restrict__ src, T *__restrict__ dst, int per_elem, int planes, int H,
                                 int W, const int *__restrict__ origins, int h, int w) {
    const int plane = blockIdx.y;
    const int n = plane / planes;
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= (int64_t)h * w * per_elem) return;
    const int64_t e = r / per_elem, k = r % per_elem;
    const int64_t y = origins[2 * n] + e / w, x = origins[2 * n + 1] + e % w;
    dst[((int64_t)plane * h * w + e) * per_elem + k] = src[(((int64_t)plane * H + y) * W + x) * per_elem + k];
}

// crop_rect_kernel with a rectangle per image, rects[n] = (y, x, h_n, w_n).  dst_off null: dst is N * planes planes of
// hp x wp, image n top-left, zero elsewhere; otherwise image n's planes of h_n x w_n start at element dst_off[n]
// (elements of per_elem words or bytes, as every other index here).
template <typename T>
__global__ void crop_rects_kernel(const T *__restrict__ src, T *__restrict__ dst, int per_elem, int planes, int H,
                                  int W, const int4 *__restrict__ rects, const int64_t *__restrict__ dst_off, int hp,
                                  int wp) {
    const int plane = blockIdx.y;
    const int n = plane / planes;
    const int4 rc = rects[n];
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t e = r / per_elem, k = r % per_elem;
    if (dst_off) {
        if (r >= (int64_t)rc.z * rc.w * per_elem) return;
        const int64_t y = rc.x + e / rc.w, x = rc.y + e % rc.w;
        dst[(dst_off[n] + (int64_t)(plane - n * planes) * rc.z * rc.w + e) * per_elem + k] =
            src[(((int64_t)plane * H + y) * W + x) * per_elem + k];
        return;
    }
    if (r >= (int64_t)hp * wp * per_elem) return;
    const int64_t oy = e / wp, ox = e % wp;
    dst[((int64_t)plane * hp * wp + e) * per_elem + k] =
        (oy < rc.z && ox < rc.w) ? src[(((int64_t)plane * H + rc.x + oy) * W + rc.y + ox) * per_elem + k] : T(0);
}

// stream order -> raster for images of different sizes: image n's planes hold the tile order of its own
// ext[n] = (h_n, w_n) plane in the first h_n * w_n of `plane_len` bytes; dst planes are hp x wp, zero outside h_n x w_n
__global__ void reorder_tiles_images_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int planes,
                                            int64_t plane_len, int hp, int wp, const int *__restrict__ ext, int th,
                                            int tw) {
    const int plane = blockIdx.y;
    const int n = plane / planes;
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= (int64_t)hp * wp) return;
    const int y = (int)(r / wp), x = (int)(r - (int64_t)y * wp), h = ext[2 * n], w = ext[2 * n + 1];
    dst[(int64_t)plane * hp * wp + r] =
        (y < h && x < w) ? src[plane * plane_len + raster_to_tile_order(y, x, h, w, th, tw)] : (uint8_t)0;
}
}  // namespace l3c

extern "C" int l3c_crop_rects(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                              const int *rects_dev, const int64_t *dst_off_dev, int hp, int wp, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(src_dev && dst_dev && src_dev != dst_dev && rects_dev, "l3c_crop_rects: bad pointers");
    L3C_REQUIRE(((uintptr_t)rects_dev & 15) == 0, "l3c_crop_rects: rects must be 16-byte aligned");
    L3C_REQUIRE(elem_bytes >= 1 && planes >= 1 && N >= 1 && (int64_t)N * planes <= 65535 && hp >= 1 && wp >= 1 &&
                    hp <= H && wp <= W,
                "l3c_crop_rects: elem_bytes=%d planes=%d N=%d %dx%d of %dx%d", elem_bytes, planes, N, hp, wp, H, W);
    const bool words = elem_bytes % 4 == 0;
    const int per_elem = words ? elem_bytes / 4 : elem_bytes;
    L3C_REQUIRE(fits_grid_x((int64_t)hp * wp, per_elem), "l3c_crop_rects: %dx%d elements of %d bytes in one launch", hp,
                wp, elem_bytes);
    dim3 grid((unsigned)ceil_div64((int64_t)hp * wp * per_elem, 256), N * planes);
    if (words)
        crop_rects_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint32_t *)src_dev, (uint32_t *)dst_dev, per_elem, planes, H, W, (const int4 *)rects_dev,
            dst_off_dev, hp, wp);
    else
        crop_rects_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint8_t *)src_dev, (uint8_t *)dst_dev, per_elem, planes, H, W, (const int4 *)rects_dev,
            dst_off_dev, hp, wp);
    L3C_LAUNCH_CHECK("crop_rects_kernel");
    return L3C_OK;
}

extern "C" int l3c_reorder_tiles_images(const uint8_t *src_dev, uint8_t *dst_dev, int planes, int N, int plane_len,
                                        int hp, int wp, const int *extents_dev, int th, int tw, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(src_dev && dst_dev && src_dev != dst_dev && extents_dev, "l3c_reorder_tiles_images: bad pointers");
    L3C_REQUIRE(planes >= 1 && N >= 1 && (int64_t)N * planes <= 65535 && hp >= 1 && wp >= 1 && th >= 1 && tw >= 1 &&
                    plane_len >= 1, "l3c_reorder_tiles_images: bad arguments");
    L3C_REQUIRE((int64_t)hp * wp < (1ll << 31), "l3c_reorder_tiles_images: %dx%d plane", hp, wp);
    dim3 grid((unsigned)ceil_div64((int64_t)hp * wp, 256), N * planes);
    reorder_tiles_images_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src_dev, dst_dev, planes, plane_len, hp, wp,
                                                                        extents_dev, th, tw);
    L3C_LAUNCH_CHECK("reorder_tiles_images_kernel");
    return L3C_OK;
}

extern "C" int l3c_crop_rect(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                             const int *origins_dev, int h, int w, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(src_dev && dst_dev && src_dev != dst_dev && origins_dev, "l3c_crop_rect: bad pointers");
    L3C_REQUIRE(elem_bytes >= 1 && planes >= 1 && N >= 1 && (int64_t)N * planes <= 65535 && h >= 1 && w >= 1 &&
                    h <= H && w <= W,
                "l3c_crop_rect: elem_bytes=%d planes=%d N=%d %dx%d of %dx%d", elem_bytes, planes, N, h, w, H, W);
    const bool words = elem_bytes % 4 == 0;
    const int per_elem = words ? elem_bytes / 4 : elem_bytes;
    L3C_REQUIRE(fits_grid_x((int64_t)h * w, per_elem), "l3c_crop_rect: %dx%d elements of %d bytes in one launch", h, w,
                elem_bytes);
    dim3 grid((unsigned)ceil_div64((int64_t)h * w * per_elem, 256), N * planes);
    if (words)
        crop_rect_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint32_t *)src_dev, (uint32_t *)dst_dev, per_elem, planes, H, W, origins_dev, h, w);
    else
        crop_rect_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint8_t *)src_dev, (uint8_t *)dst_dev, per_elem, planes, H, W, origins_dev, h, w);
    L3C_LAUNCH_CHECK("crop_rect_kernel");
    return L3C_OK;
}

extern "C" int l3c_reorder_tiles(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int H, int W, int th,
                                 int tw, int to_tiles, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(src_dev && dst_dev && src_dev != dst_dev, "l3c_reorder_tiles: bad pointers");
    L3C_REQUIRE((elem_bytes == 1 || elem_bytes == 4) && planes >= 1 && planes <= 65535 && H >= 1 && W >= 1 && th >= 1 &&
                    tw >= 1, "l3c_reorder_tiles: bad arguments");
    L3C_REQUIRE((int64_t)H * W < (1ll << 31), "l3c_reorder_tiles: %dx%d plane", H, W);
    // a tile that reaches past the plane is the plane's extent in that direction: the same order, and the tile
    // arithmetic (th * W, tw * th) stays below H * W
    th = th < H ? th : H;
    tw = tw < W ? tw : W;
    const int HW = H * W;
    dim3 grid((unsigned)ceil_div64(HW, 256), planes);
    if (elem_bytes == 1)
        reorder_tiles_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src_dev, (uint8_t *)dst_dev,
                                                                              HW, H, W, th, tw, to_tiles);
    else
        reorder_tiles_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint32_t *)src_dev,
                                                                               (uint32_t *)dst_dev, HW, H, W, th, tw, to_tiles);
    L3C_LAUNCH_CHECK("reorder_tiles_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_nll(const float *l_dev, const uint8_t *sym_dev, const float *values_dev,
                            int N, int HW, int C, int K, int L, int rgb, float x_min, float x_max,
                            double *nll_dev, float *nll_map_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_nll", N, HW, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && sym_dev && values_dev && nll_dev, "l3c_dmll_nll: null pointer");
    const int per_image = ceil_div(HW, NLL_THREADS);
    double *partial = nullptr;
    L3C_CUDA(cudaMallocAsync(&partial, sizeof(double) * (size_t)N * per_image, (cudaStream_t)stream));
    dim3 grid(per_image, N);                                 // the plane as one row of HW pixels
    dmll_nll_kernel<10, false><<<grid, NLL_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, values_dev, 1, HW, C, L, rgb, x_min, x_max, nullptr, partial, nll_map_dev);
    L3C_LAUNCH_CHECK("dmll_nll_kernel");
    nll_finish_kernel<<<N, 32, 0, (cudaStream_t)stream>>>(partial, per_image, 1, HW, nullptr, nll_dev);
    L3C_LAUNCH_CHECK("nll_finish_kernel");
    L3C_CUDA(cudaFreeAsync(partial, (cudaStream_t)stream));
    return L3C_OK;
}

extern "C" int l3c_dmll_nll_ragged(const float *l_dev, const uint8_t *sym_dev, const float *values_dev, int N, int H,
                                   int W, int C, int K, int L, int rgb, float x_min, float x_max,
                                   const int *extents_dev, double *nll_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(H >= 1 && W >= 1 && (int64_t)H * W <= INT32_MAX, "l3c_dmll_nll_ragged: H=%d W=%d", H, W);
    if (int e = check_common("l3c_dmll_nll_ragged", N, H * W, C, K, L, rgb)) return e;
    L3C_REQUIRE(l_dev && sym_dev && values_dev && extents_dev && nll_dev, "l3c_dmll_nll_ragged: null pointer");
    // CTAs for the largest image the plane can hold; those beyond an image's own pixels exit at once
    const int per_image = ceil_div(H * W, NLL_THREADS);
    double *partial = nullptr;
    L3C_CUDA(cudaMallocAsync(&partial, sizeof(double) * (size_t)N * per_image, (cudaStream_t)stream));
    dim3 grid(per_image, N);
    dmll_nll_kernel<10, true><<<grid, NLL_THREADS, 0, (cudaStream_t)stream>>>(
        l_dev, sym_dev, values_dev, H, W, C, L, rgb, x_min, x_max, extents_dev, partial, nullptr);
    L3C_LAUNCH_CHECK("dmll_nll_kernel");
    nll_finish_kernel<<<N, 32, 0, (cudaStream_t)stream>>>(partial, per_image, H, W, extents_dev, nll_dev);
    L3C_LAUNCH_CHECK("nll_finish_kernel");
    L3C_CUDA(cudaFreeAsync(partial, (cudaStream_t)stream));
    return L3C_OK;
}

extern "C" int l3c_dmll_nll_train(const float *l_dev, const float *x_dev, int N, int HW, int C, int K, int rgb,
                                  float half_bin, float x_lower, float x_upper, double *nll_dev,
                                  const float *grad_dev, float *dl_dev, float *dx_dev, void *stream) {
    using namespace l3c;
    // the alphabet does not enter the loss (the targets are values, the bin width comes as half_bin): any L passes
    if (int e = check_common("l3c_dmll_nll_train", N, HW, C, K, 256, rgb)) return e;
    L3C_REQUIRE(l_dev && x_dev, "l3c_dmll_nll_train: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int per_image = ceil_div(HW, NLL_THREADS);
    dim3 grid(per_image, N);
    if (grad_dev) {
        L3C_REQUIRE(dl_dev, "l3c_dmll_nll_train: the backward needs dl_dev");
        L3C_REQUIRE(!(rgb && dx_dev), "l3c_dmll_nll_train: no dx at an RGB scale (the image is not differentiable)");
        dmll_train_grad_kernel<10><<<grid, NLL_THREADS, 0, st>>>(l_dev, x_dev, HW, C, rgb, half_bin, x_lower, x_upper,
                                                                 grad_dev, dl_dev, dx_dev);
        L3C_LAUNCH_CHECK("dmll_train_grad_kernel");
        return L3C_OK;
    }
    L3C_REQUIRE(nll_dev, "l3c_dmll_nll_train: the forward needs nll_dev");
    double *partial = nullptr;
    L3C_CUDA(cudaMallocAsync(&partial, sizeof(double) * (size_t)N * per_image, st));
    dmll_train_nll_kernel<10><<<grid, NLL_THREADS, 0, st>>>(l_dev, x_dev, HW, C, rgb, half_bin, x_lower, x_upper,
                                                            partial);
    L3C_LAUNCH_CHECK("dmll_train_nll_kernel");
    nll_finish_kernel<<<N, 32, 0, st>>>(partial, per_image, 1, HW, nullptr, nll_dev);
    L3C_LAUNCH_CHECK("nll_finish_kernel");
    L3C_CUDA(cudaFreeAsync(partial, st));
    return L3C_OK;
}

extern "C" int l3c_soft_quantize(const float *q_dev, int64_t n, const float *levels_dev, int L, float sigma,
                                 int64_t *sym_dev, float *value_dev, const float *grad_dev, float *dq_dev,
                                 void *stream) {
    using namespace l3c;
    L3C_REQUIRE(q_dev && levels_dev && n >= 0, "l3c_soft_quantize: bad arguments");
    L3C_REQUIRE(L >= 1 && L <= 256, "l3c_soft_quantize: L=%d", L);
    L3C_REQUIRE(grad_dev ? (dq_dev != nullptr) : (sym_dev && value_dev),
                "l3c_soft_quantize: the forward needs sym_dev and value_dev, the backward dq_dev");
    L3C_REQUIRE(!grad_dev || sigma > 0.f, "l3c_soft_quantize: sigma=%g must be positive", (double)sigma);
    L3C_REQUIRE(ceil_div64(n, SQ_THREADS) <= INT32_MAX, "l3c_soft_quantize: n=%lld", (long long)n);
    if (n == 0) return L3C_OK;
    soft_quantize_kernel<<<(unsigned)ceil_div64(n, SQ_THREADS), SQ_THREADS, L * sizeof(float), (cudaStream_t)stream>>>(
        q_dev, n, levels_dev, L, sigma, sym_dev, value_dev, grad_dev, dq_dev);
    L3C_LAUNCH_CHECK("soft_quantize_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_channel_params(const float *l_dev, const float *x_dec_dev, int N, int HW,
                                       int C, int K, int rgb, int c, float *pi_dev, float *mu_dev,
                                       float *log_scales_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_channel_params", N, HW, C, K, 256, rgb)) return e;
    L3C_REQUIRE(l_dev && pi_dev && mu_dev && log_scales_dev && c >= 0 && c < C,
                "l3c_dmll_channel_params: bad arguments");
    L3C_REQUIRE(!(rgb && c > 0) || x_dec_dev, "l3c_dmll_channel_params: decoded values needed for c>0");
    dim3 grid(ceil_div(HW, 128), N);
    dmll_channel_params_kernel<10><<<grid, 128, 0, (cudaStream_t)stream>>>(
        l_dev, x_dec_dev, HW, C, rgb, c, pi_dev, mu_dev, log_scales_dev);
    L3C_LAUNCH_CHECK("dmll_channel_params_kernel");
    return L3C_OK;
}

extern "C" int l3c_dmll_sample(const float *l_dev, const float *u_sel_dev, const float *u_x_dev, int N, int HW,
                               int C, int K, int rgb, float *x_dev, void *stream) {
    using namespace l3c;
    if (int e = check_common("l3c_dmll_sample", N, HW, C, K, 256, rgb)) return e;
    L3C_REQUIRE(l_dev && u_sel_dev && u_x_dev && x_dev, "l3c_dmll_sample: null pointer");
    dim3 grid(ceil_div(HW, 128), N);
    dmll_sample_kernel<10><<<grid, 128, 0, (cudaStream_t)stream>>>(l_dev, u_sel_dev, u_x_dev, HW, C, rgb, x_dev);
    L3C_LAUNCH_CHECK("dmll_sample_kernel");
    return L3C_OK;
}

namespace l3c {
// the sigmoid of the CDF rows and one saturating mixture term (pi = 1, acc = 0), through the same __device__
// functions every CDF kernel calls
__global__ void probe_sigmoid_kernel(const float *__restrict__ u, float *__restrict__ raw, float *__restrict__ term,
                                     int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = u[i];
        raw[i] = sigmoid_from_log2(v);
        term[i] = mixture_term(0.f, 1.f, v);
    }
}
}  // namespace l3c

extern "C" int l3c_dmll_probe_sigmoid(const float *u_dev, float *raw_dev, float *term_dev, int64_t n, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(u_dev && raw_dev && term_dev && n >= 0, "l3c_dmll_probe_sigmoid: bad arguments");
    if (n == 0) return L3C_OK;
    const int64_t want = ceil_div64(n, 256);
    const int blocks = (int)(want < 65536 ? want : 65536);
    probe_sigmoid_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(u_dev, raw_dev, term_dev, n);
    L3C_LAUNCH_CHECK("probe_sigmoid_kernel");
    return L3C_OK;
}
