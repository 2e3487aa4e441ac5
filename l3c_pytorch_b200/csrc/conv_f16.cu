// conv_f16.cu -- precision mode L3C_PREC_F16: the 64-input-channel 3x3 (optionally dilated) layers, the 5x5/s2
// down-sampling layers and the 1x1 layers of the L3C stack as implicit GEMMs on the Hopper tensor cores with FP16
// operands (wgmma m64n64k16) and fp32 accumulation in registers.
//
// Reference layers this replaces: every `default_conv(64, Cout, 3, rate=r)` of the stack
// (pytorch_ext.py:57-61; ResBlock edsr.py:63-89, body-final conv net.py:110,170, Head head.py:49-56,
// Upsampler edsr.py:92-101, atrous convs prob_clf.py:54-55) and the 1x1 `lin` conv of the probability
// classifier (prob_clf.py:56,71-74) -- cuDNN fp32 in the reference.
//
// Why FP16 operands.  Round-to-nearest FP16 keeps the same 10 explicit mantissa bits as the TF32-RN operands of
// conv_tf32.cu (identical values for 6.1e-5 <= |x| <= 65504; saturating conversion above, absolute error < 3e-8
// below), but
//   * one wgmma covers K = 16 instead of 8 at twice the TF32 rate;
//   * an activation's operand image is 128 B per pixel (64 channels) = exactly ONE 128B-swizzle row, so a halo
//     box needs one TMA load per filter column (no K-halves) and half the L2->smem bytes;
//   * operand twins cost 128 instead of 256 B per pixel in HBM, and a layer whose output only feeds tensor-core
//     convs (first conv of a ResBlock, atrous convs, the finest decoder features) writes ONLY the 2-byte image.
// Per pixel a 64->64 conv moves 256 B (operand in / operand out) to 768 B (operand + fp32 residual in, fp32 +
// operand out) against 73.7 kFLOP.
//
// Structure of the 3x3 kernel (persistent, tc_ptx.cuh layout: two consumer warpgroups with a TMA producer warp
// each):
//   * the 9 weight slabs of the CTA's Cout tile (9 x 64 rows x 128 B = 72 KB) stay in shared memory;
//   * per filter column dx ONE box of (8 + 2d) rows x 16 pixels x 64 channels is staged by TMA; the three dy taps
//     read it at row offsets dy*d*2048 B (multiples of the 1024 B swizzle atom);
//   * the consumer warpgroup accumulates the two 64-pixel halves of the 8x16 tile (2 x 32 registers per
//     thread), then fuses bias / ReLU / residual / PixelShuffle(2), writes fp32 float2 (full sectors) and the FP16
//     image as 16-byte vectors after a 4x4 transpose inside each quad.
// Accumulation order per output element: (dx, dy, k-step) -- fixed, independent of batch / image size / tile
// position / pipe: encoder-side and decoder-side evaluations are bit-identical.
#include <cuda.h>
#include <stdlib.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "dmll_math.cuh"

namespace l3c {
namespace f16 {
using namespace tcx;

constexpr int TH = 8, TW = 16;                 // 128 output pixels per tile
constexpr int W_TAP_BYTES = 64 * 128;          // one filter tap of one Cout tile: 64 rows x 64 fp16
constexpr int W_RES_BYTES = 9 * W_TAP_BYTES;   // 73728
constexpr int MAX_STAGES = 4;
constexpr int BARS_PER_PIPE = 2 * MAX_STAGES;  // full[4], empty[4]

struct Params {
    const float *bias;      // padded to cout_pad
    const float *residual;  // fp32, layout of y, or null
    float *y;               // fp32 output or null
    __half *yh;             // fp16 operand image of the output or null
    int N, H, W;
    int Cout, y_pitch, y_coff;
    int dilation;
    unsigned flags;
    int tiles_x, tiles_y;
};

// two floats -> packed fp16 pair, round-to-nearest-even, saturating to +-65504
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // d.hi = first source
    return r;
}
constexpr float LO_INV = 1.0f / 2048.0f;       // precision mode f16x2: x = hi + lo / 2^11

// 4x4 transpose inside each quad of lanes: before, thread tq holds v[j] = element (column block j, pair tq);
// after, thread tq holds v[s] = element (column block tq, pair s) -> 8 consecutive channels = 16 bytes.
// Must be executed by all 32 lanes.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int tq) {
    const bool hi2 = (tq & 2) != 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const uint32_t send = hi2 ? v[i] : v[i + 2];
        const uint32_t got = __shfl_xor_sync(0xFFFFFFFFu, send, 2);
        if (hi2) v[i] = got; else v[i + 2] = got;
    }
    const bool hi1 = (tq & 1) != 0;
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
        const uint32_t send = hi1 ? v[i] : v[i + 1];
        const uint32_t got = __shfl_xor_sync(0xFFFFFFFFu, send, 1);
        if (hi1) v[i] = got; else v[i + 1] = got;
    }
}

// KIND 0: 3x3 stride 1 (any dilation), weights resident.
// KIND 1: 5x5 stride 2 (the down-sampling conv of every encoder, net.py:101): the input box of a tap is read
//   with TMA element strides (2, 2), so the A operand of an 8x16 OUTPUT tile is again 128 dense rows of 128 B;
//   for a filter column kx the taps ky = 0,2,4 (and ky = 1,3) share one strided box of 10 rows read at row
//   offsets j*2048 B.  25 taps x 8 KB of weights do not fit beside the stages: every unit (kx, row parity)
//   brings its 3 (2) weight slabs along with its box.  10 units, 100 k-steps per tile.
constexpr int K5_A_BYTES = 10 * TW * 128;                  // 20480: strided halo box
constexpr int K5_STAGE_BYTES = K5_A_BYTES + 3 * W_TAP_BYTES;   // 45056: box + up to three weight slabs

template <int KIND>
__global__ void __launch_bounds__(THREADS, 1)
conv_f16_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                const Params p, const int n_stages, const int a_bytes, const int ptiles) {
    constexpr int W_RES = (KIND == 0) ? W_RES_BYTES : 0;    // resident weights
    constexpr int UNITS = (KIND == 0) ? 3 : 10;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    // [weights 72 KB][pipe 0 stages][pipe 1 stages][barriers]
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + W_RES + 2 * n_stages * a_bytes);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t w_base = smem_u32(smem);
    const uint32_t bar_base = smem_u32(bars);
    const uint32_t wbar = bar_base + 8u * (2 * BARS_PER_PIPE);

    if (threadIdx.x == 0) {
        for (int k = 0; k < 2; ++k)
            for (int s = 0; s < MAX_STAGES; ++s) {
                mbar_init(bar_base + 8u * (BARS_PER_PIPE * k + s), 1);                  // full
                mbar_init(bar_base + 8u * (BARS_PER_PIPE * k + MAX_STAGES + s), 4);     // empty: one per consumer warp
            }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    }
    __syncthreads();

    const int d = p.dilation;
    const int ct = blockIdx.y;                        // this CTA's Cout tile (weights stay resident)

    if (warp >= CONSUMER_WARPS) {
        // ===================== TMA producer of pipe k =====================
        const int k = warp - CONSUMER_WARPS;
        if (lane != 0) return;
        const uint32_t a_base = w_base + W_RES + k * n_stages * a_bytes;
        const uint32_t full0 = bar_base + 8u * (BARS_PER_PIPE * k), empty0 = full0 + 8u * MAX_STAGES;
        if (KIND == 0 && k == 0) {
            mbar_expect_tx(wbar, W_RES_BYTES);
            for (int tap = 0; tap < 9; ++tap)         // rows [tap][cout_pad] of the weight image
                tma_load_2d(w_base + tap * W_TAP_BYTES, &map_w, wbar, 0, tap * (int)gridDim.y * 64 + ct * 64);
        }
        uint32_t stage = 0, phase = 0;
        for (int t = blockIdx.x + k * gridDim.x; t < ptiles; t += 2 * gridDim.x) {
            int q = t;
            const int tx = q % p.tiles_x; q /= p.tiles_x;
            const int ty = q % p.tiles_y; q /= p.tiles_y;
            const int n = q;
            for (int u = 0; u < UNITS; ++u) {
                mbar_wait(empty0 + 8u * stage, phase ^ 1u);
                const uint32_t dst = a_base + stage * a_bytes, bar = full0 + 8u * stage;
                if (KIND == 0) {
                    mbar_expect_tx(bar, a_bytes);
                    tma_load_4d(dst, &map_x, bar, 0, tx * TW + (u - 1) * d, ty * TH - d, n);
                } else {
                    const int kx = u >> 1, par = u & 1, ntaps = 3 - par;
                    mbar_expect_tx(bar, K5_A_BYTES + ntaps * W_TAP_BYTES);
                    // input pixel of output (oy, ox), tap (ky, kx): (2*oy + ky - 2, 2*ox + kx - 2)
                    tma_load_4d(dst, &map_x, bar, 0, 2 * tx * TW + kx - 2, 2 * ty * TH + par - 2, n);
                    for (int j = 0; j < ntaps; ++j)
                        tma_load_2d(dst + K5_A_BYTES + j * W_TAP_BYTES, &map_w, bar, 0,
                                    ((par + 2 * j) * 5 + kx) * (int)gridDim.y * 64 + ct * 64);
                }
                if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }

    // ===================== consumer warpgroup k: wgmma + epilogue =====================
    const int k = warp >> 2, w = warp & 3;
    const uint32_t a_base = w_base + W_RES + k * n_stages * a_bytes;
    const uint32_t full0 = bar_base + 8u * (BARS_PER_PIPE * k), empty0 = full0 + 8u * MAX_STAGES;
    const int tq = lane & 3, tr = lane >> 2;              // column pair / row inside the fragment
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool shuffle = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
    uint32_t stage = 0, phase = 0;
    if (KIND == 0) mbar_wait(wbar, 0);
    for (int t = blockIdx.x + k * gridDim.x; t < ptiles; t += 2 * gridDim.x) {
        int q = t;
        const int tx = q % p.tiles_x; q /= p.tiles_x;
        const int ty = q % p.tiles_y; q /= p.tiles_y;
        const int n = q;
        float acc[2][32];                                 // rows 0..63 / 64..127 of the tile
        acc_zero(acc[0]);
        acc_zero(acc[1]);
        for (int u = 0; u < UNITS; ++u) {
            mbar_wait(full0 + 8u * stage, phase);
            const uint32_t a0 = a_base + stage * a_bytes;
            wgmma_fence();
            if (KIND == 0) {
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    const uint64_t db = make_desc(w_base + (dy * 3 + u) * W_TAP_BYTES);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint64_t da = make_desc(a0 + (dy * d * TW + 64 * h) * 128);   // dy*d rows of 16 px
#pragma unroll
                        for (int kk = 0; kk < 4; ++kk)                                       // +32 B = 16 fp16 along K
                            wgmma_f16(acc[h], da + 2u * kk, db + 2u * kk, (u | dy | kk) != 0 ? 1u : 0u);
                    }
                }
            } else {
                const int ntaps = 3 - (u & 1);
                for (int j = 0; j < ntaps; ++j) {
                    const uint64_t db = make_desc(a0 + K5_A_BYTES + j * W_TAP_BYTES);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint64_t da = make_desc(a0 + (j * TW + 64 * h) * 128);        // box row j = tap ky0 + 2j
#pragma unroll
                        for (int kk = 0; kk < 4; ++kk)
                            wgmma_f16(acc[h], da + 2u * kk, db + 2u * kk, (u | j | kk) != 0 ? 1u : 0u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait0();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + 8u * stage);      // frees the stage for the producer
            if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
        }
        // epilogue: fragment (h, column half c) = tile row 4h + w, pixels tr / tr + 8, columns 32c + 8jb + 2tq
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int oy = ty * TH + 4 * h + w;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const float *v = acc[h] + 16 * c;
                const int cb = ct * 64 + 32 * c;                      // first conv channel of this fragment
#pragma unroll
                for (int rh = 0; rh < 2; ++rh) {
                    const int ox = tx * TW + tr + 8 * rh;
                    const bool inside = (oy < p.H) && (ox < p.W);
                    const size_t pix = ((size_t)n * p.H + oy) * p.W + ox;
                    float a[4], b[4];
#pragma unroll
                    for (int jb = 0; jb < 4; ++jb) {
                        const float2 bb = __ldg(reinterpret_cast<const float2 *>(p.bias + cb + 8 * jb + 2 * tq));
                        a[jb] = v[4 * jb + 2 * rh] + bb.x;
                        b[jb] = v[4 * jb + 2 * rh + 1] + bb.y;
                        if (relu) { a[jb] = fmaxf(a[jb], 0.f); b[jb] = fmaxf(b[jb], 0.f); }
                    }
                    if (!shuffle) {
                        const size_t off = pix * p.y_pitch + p.y_coff + cb;
                        if (p.residual != nullptr && inside) {
#pragma unroll
                            for (int jb = 0; jb < 4; ++jb) {
                                const float2 r = __ldg(reinterpret_cast<const float2 *>(p.residual + off + 8 * jb + 2 * tq));
                                a[jb] += r.x; b[jb] += r.y;
                            }
                        }
                        if (p.y != nullptr && inside) {
#pragma unroll
                            for (int jb = 0; jb < 4; ++jb)
                                *reinterpret_cast<float2 *>(p.y + off + 8 * jb + 2 * tq) = make_float2(a[jb], b[jb]);
                        }
                        if (p.yh != nullptr) {
                            uint32_t hv[4];
#pragma unroll
                            for (int jb = 0; jb < 4; ++jb) hv[jb] = pack_h2(a[jb], b[jb]);
                            quad_transpose(hv, tq);           // -> channels cb + 8*tq + 0..7
                            if (inside) *reinterpret_cast<uint4 *>(p.yh + off + 8 * tq) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
                        }
                    } else {
                        // out[n, 2*oy+si, 2*ox+sj, cq] = conv[n, oy, ox, 4*cq + 2*si + sj]   (edsr.py:92-101)
                        const size_t W2 = 2 * (size_t)p.W;
                        const size_t row0 = ((size_t)n * (2 * p.H) + 2 * oy) * W2 + 2 * ox;   // output pixel (si=0, sj=0)
                        if (p.y != nullptr) {
                            // same transpose on the fp32 values: thread tq then owns conv channels c0 + 0..7
                            // (c0 = cb + 8*tq) = output channels cq0, cq0 + 1 of the four sub-pixels, and a quad
                            // writes 32 contiguous bytes per output pixel
                            uint32_t fa[4], fb[4];
#pragma unroll
                            for (int jb = 0; jb < 4; ++jb) { fa[jb] = __float_as_uint(a[jb]); fb[jb] = __float_as_uint(b[jb]); }
                            quad_transpose(fa, tq);           // fa[s] = channel c0 + 2s, fb[s] = channel c0 + 2s + 1
                            quad_transpose(fb, tq);
                            if (inside) {
                                const int cq0 = (cb + 8 * tq) >> 2;
#pragma unroll
                                for (int si = 0; si < 2; ++si) {
                                    const size_t o2 = (row0 + si * W2) * p.y_pitch + p.y_coff + cq0;
                                    *reinterpret_cast<float2 *>(p.y + o2) =
                                        make_float2(__uint_as_float(fa[si]), __uint_as_float(fa[2 + si]));        // sj = 0
                                    *reinterpret_cast<float2 *>(p.y + o2 + p.y_pitch) =
                                        make_float2(__uint_as_float(fb[si]), __uint_as_float(fb[2 + si]));        // sj = 1
                                }
                            }
                        }
                        if (p.yh != nullptr) {
                            uint32_t hv[4];
#pragma unroll
                            for (int jb = 0; jb < 4; ++jb) hv[jb] = pack_h2(a[jb], b[jb]);
                            quad_transpose(hv, tq);           // hv[s] = conv channels c0 + 2s + {0,1}, c0 = cb + 8*tq
                            if (inside) {
                                const int cq0 = (cb + 8 * tq) >> 2;          // output channels cq0, cq0 + 1
#pragma unroll
                                for (int si = 0; si < 2; ++si) {
                                    const size_t o2 = (row0 + si * W2) * p.y_pitch + p.y_coff + cq0;
                                    // sj = 0: low halves of hv[si] (cq0) and hv[2+si] (cq0+1); sj = 1: the high halves
                                    *reinterpret_cast<uint32_t *>(p.yh + o2) = __byte_perm(hv[si], hv[2 + si], 0x5410);
                                    *reinterpret_cast<uint32_t *>(p.yh + o2 + p.y_pitch) = __byte_perm(hv[si], hv[2 + si], 0x7632);
                                }
                            }
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 1x1 layers (Cin % 64 == 0, e.g. the 192 -> Kp `lin` conv of the probability classifier, the im2col GEMM of the
// RGB head) in all three tensor-core precisions: a plain GEMM [pixels][Cin] x [Cin][Cout].  Tile = 64 consecutive
// pixels x NB blocks of 64 output channels (all of them unless the split mode's two accumulators would not fit in
// registers), the two consumer warpgroups take alternate tiles; the weights (K chunks x cout_pad rows x 128 B, two
// planes in mode f16x2) stay in shared memory.  HBM-bound: per pixel the operand row in, 4*Cout bytes out.
//   KIND 0 (tf32):  K chunk = 32 fp32 channels; weight image [Cin/32][cout_pad][32] fp32; fp32 + TF32 twin out
//   KIND 1 (f16):   K chunk = 64 fp16 channels; weight image [Cin/64][cout_pad][64]; fp32 and / or FP16 image out
//   KIND 2 (f16x2): K chunk = 64 channels of the hi and of the lo plane; weights [2*Cin/64][cout_pad][64];
//                   acc1 += hi*hi, acc2 += hi*lo + lo*hi; fp32 out
// ---------------------------------------------------------------------------------------------
constexpr int K1_A_BYTES = 64 * 128;           // one K chunk of a 64-pixel tile
constexpr int K1_MAX_STAGES = 4;

struct Params1 {
    const float *bias;
    const float *residual;   // KIND 0 only
    float *y;
    float *y_tf32;           // KIND 0 only
    __half *yh;              // KIND 1 only
    long long M;             // pixels
    int Cout, y_pitch, y_coff;
    unsigned flags;
    int kunits, npad, lo_ch, nch;   // K chunks, cout_pad, lo plane offset (KIND 2), Cout chunks per pixel tile
};

template <int KIND, int NB>
__global__ void __launch_bounds__(THREADS, 1)
conv1x1_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                  const Params1 p, const int n_stages, const int n_tiles) {
    constexpr int PLANES = (KIND == 2) ? 2 : 1;
    constexpr int SB = PLANES * K1_A_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int w_plane = p.kunits * p.npad * 128;
    // [weights (hi plane, lo plane)][pipe 0 stages][pipe 1 stages][barriers: per pipe full[4], empty[4]; weights]
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + PLANES * w_plane + 2 * n_stages * SB);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t w_base = smem_u32(smem);
    const uint32_t bar_base = smem_u32(bars);
    const uint32_t wbar = bar_base + 8u * (4 * K1_MAX_STAGES);

    if (threadIdx.x == 0) {
        for (int k = 0; k < 2; ++k)
            for (int s = 0; s < K1_MAX_STAGES; ++s) {
                mbar_init(bar_base + 8u * (2 * K1_MAX_STAGES * k + s), 1);
                mbar_init(bar_base + 8u * (2 * K1_MAX_STAGES * k + K1_MAX_STAGES + s), 4);
            }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    }
    __syncthreads();

    if (warp >= CONSUMER_WARPS) {
        // ===================== TMA producer of pipe k =====================
        const int k = warp - CONSUMER_WARPS;
        if (lane != 0) return;
        const uint32_t a_base = w_base + PLANES * w_plane + k * n_stages * SB;
        const uint32_t full0 = bar_base + 8u * (2 * K1_MAX_STAGES * k), empty0 = full0 + 8u * K1_MAX_STAGES;
        constexpr int CH = (KIND == 0) ? 32 : 64;           // channels per K chunk
        if (k == 0) {
            mbar_expect_tx(wbar, (uint32_t)(PLANES * w_plane));
            for (int kc = 0; kc < PLANES * p.kunits; ++kc)
                tma_load_2d(w_base + kc * p.npad * 128, &map_w, wbar, 0, kc * p.npad);
        }
        uint32_t stage = 0, phase = 0;
        for (int t = blockIdx.x + k * gridDim.x; t < n_tiles; t += 2 * gridDim.x) {
            const int pt = t / p.nch;
            for (int u = 0; u < p.kunits; ++u) {
                mbar_wait(empty0 + 8u * stage, phase ^ 1u);
                const uint32_t dst = a_base + stage * SB, bar = full0 + 8u * stage;
                mbar_expect_tx(bar, SB);
                tma_load_2d(dst, &map_x, bar, u * CH, pt * 64);
                if (KIND == 2) tma_load_2d(dst + K1_A_BYTES, &map_x, bar, p.lo_ch + u * CH, pt * 64);
                if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }

    // ===================== consumer warpgroup k =====================
    const int k = warp >> 2, w = warp & 3;
    const uint32_t a_base = w_base + PLANES * w_plane + k * n_stages * SB;
    const uint32_t full0 = bar_base + 8u * (2 * K1_MAX_STAGES * k), empty0 = full0 + 8u * K1_MAX_STAGES;
    const int tq = lane & 3, tr = lane >> 2;
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool round_y = (p.flags & L3C_CONV_ROUND_TF32) != 0;
    uint32_t stage = 0, phase = 0;
    mbar_wait(wbar, 0);
    for (int t = blockIdx.x + k * gridDim.x; t < n_tiles; t += 2 * gridDim.x) {
        const int pt = t / p.nch, nc = t % p.nch;
        float acc[NB][32], acc2[NB][32];          // acc2: KIND 2 only
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) acc_zero(acc[nb]);
        if (KIND == 2) {
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) acc_zero(acc2[nb]);
        }
        for (int u = 0; u < p.kunits; ++u) {
            mbar_wait(full0 + 8u * stage, phase);
            const uint32_t a0 = a_base + stage * SB;
            wgmma_fence();
            const uint64_t ah = make_desc(a0);
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
                const int col = (nc * NB + nb) * 64;
                const uint64_t bh = make_desc(w_base + (u * p.npad + col) * 128);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const uint32_t first = (u | kk) != 0 ? 1u : 0u;
                    if (KIND == 0) {
                        wgmma_tf32(acc[nb], ah + 2u * kk, bh + 2u * kk, first);
                    } else {
                        wgmma_f16(acc[nb], ah + 2u * kk, bh + 2u * kk, first);
                        if (KIND == 2) {
                            const uint64_t al = make_desc(a0 + K1_A_BYTES);
                            const uint64_t bl = make_desc(w_base + w_plane + (u * p.npad + col) * 128);
                            wgmma_f16(acc2[nb], ah + 2u * kk, bl + 2u * kk, first);   // hi * lo
                            wgmma_f16(acc2[nb], al + 2u * kk, bh + 2u * kk, 1u);      // lo * hi
                        }
                    }
                }
            }
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) acc_fence(acc[nb]);
            if (KIND == 2) {
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) acc_fence(acc2[nb]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + 8u * stage);
            if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
        }
        // epilogue: pixel pt*64 + 16w + tr + 8rh, channels (nc*NB + nb)*64 + 8j + 2tq + {0,1}
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
            const long long pix = (long long)pt * 64 + 16 * w + tr + 8 * rh;
            if (pix >= p.M) continue;
            const size_t off = (size_t)pix * p.y_pitch + p.y_coff;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int co = (nc * NB + nb) * 64 + 8 * j + 2 * tq;
                    if (co >= p.Cout) continue;
                    const float2 bb = __ldg(reinterpret_cast<const float2 *>(p.bias + co));   // padded to cout_pad
                    float a = acc[nb][4 * j + 2 * rh], b = acc[nb][4 * j + 2 * rh + 1];
                    if (KIND == 2) {
                        a = __fmaf_rn(acc2[nb][4 * j + 2 * rh], LO_INV, a);
                        b = __fmaf_rn(acc2[nb][4 * j + 2 * rh + 1], LO_INV, b);
                    }
                    a += bb.x;
                    b += bb.y;
                    if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                    if (KIND == 0) {
                        // any Cout and pitch: element stores, the second channel guarded
                        const bool two = co + 1 < p.Cout;
                        if (p.residual) {
                            a += __ldg(p.residual + off + co);
                            if (two) b += __ldg(p.residual + off + co + 1);
                        }
                        if (p.y_tf32) {
                            p.y_tf32[off + co] = round_tf32(a);
                            if (two) p.y_tf32[off + co + 1] = round_tf32(b);
                        }
                        if (round_y) { a = round_tf32(a); b = round_tf32(b); }
                        p.y[off + co] = a;
                        if (two) p.y[off + co + 1] = b;
                    } else {
                        // Cout, pitch and offset are even
                        if (p.y != nullptr) *reinterpret_cast<float2 *>(p.y + off + co) = make_float2(a, b);
                        if (KIND == 1 && p.yh != nullptr) *reinterpret_cast<uint32_t *>(p.yh + off + co) = pack_h2(a, b);
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// The DMLL head fused into the 1x1 `lin` conv of the probability classifier (encode side): the GEMM of
// conv1x1_tc_kernel<1, NB> (all npad = NB*64 channels per 64-pixel tile), but the epilogue never writes the Kp
// parameters of a pixel (480 / 600 B) to HBM -- the warpgroup parks its accumulators in shared memory, and then
// each thread owns one (pixel, channel parity) pair, reads the K logits / means / log-scales (and RGB coefficients)
// of one channel at a time, and evaluates the two CDF bounds of the symbol being coded (dmll_math.cuh: the SAME
// functions the decoder's row builder uses on the parameters it computes with the plain kernel, so both sides see
// identical integers).  Output: 4 B per coded sub-pixel.
// Reference: criterion/logistic_mixture.py:248-275 + torchac_kernel.cu:26-76 after prob_clf.py:71-74.
// ---------------------------------------------------------------------------------------------
struct ParamsLD {
    const float *bias;
    const uint8_t *sym;         // [N][C][HW] symbols being coded
    const float *targets;       // [L + 1] bin edges
    uint32_t *intervals;        // [N][C][HW] out
    long long M;                // pixels = N * HW
    int HW, L;
    int kchunks, npad;
};

template <int C, bool RGB, int NB>
__global__ void __launch_bounds__(THREADS, 1)
lin_dmll_f16_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const ParamsLD p, const int n_stages, const int n_tiles) {
    constexpr int K = 10;
    constexpr int KP = (RGB ? 4 : 3) * C * K;            // parameters per pixel (the bias has KP entries)
    constexpr int NPAD = NB * 64, S = NPAD + 1;         // staging row pitch (floats): conflict-free column reads
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int w_bytes = p.kchunks * NPAD * 128;
    // [weights][pipe 0 stages][pipe 1 stages][staging 2 x 64 x S fp32][barriers]
    float *staging = reinterpret_cast<float *>(smem + w_bytes + 2 * n_stages * K1_A_BYTES);
    uint64_t *bars = reinterpret_cast<uint64_t *>(staging + 2 * 64 * S);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t w_base = smem_u32(smem);
    const uint32_t bar_base = smem_u32(bars);
    const uint32_t wbar = bar_base + 8u * (4 * K1_MAX_STAGES);

    if (threadIdx.x == 0) {
        for (int k = 0; k < 2; ++k)
            for (int s = 0; s < K1_MAX_STAGES; ++s) {
                mbar_init(bar_base + 8u * (2 * K1_MAX_STAGES * k + s), 1);
                mbar_init(bar_base + 8u * (2 * K1_MAX_STAGES * k + K1_MAX_STAGES + s), 4);
            }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    }
    __syncthreads();

    if (warp >= CONSUMER_WARPS) {
        const int k = warp - CONSUMER_WARPS;
        if (lane != 0) return;
        const uint32_t a_base = w_base + w_bytes + k * n_stages * K1_A_BYTES;
        const uint32_t full0 = bar_base + 8u * (2 * K1_MAX_STAGES * k), empty0 = full0 + 8u * K1_MAX_STAGES;
        if (k == 0) {
            mbar_expect_tx(wbar, (uint32_t)w_bytes);
            for (int kc = 0; kc < p.kchunks; ++kc)
                tma_load_2d(w_base + kc * NPAD * 128, &map_w, wbar, 0, kc * NPAD);
        }
        uint32_t stage = 0, phase = 0;
        for (int t = blockIdx.x + k * gridDim.x; t < n_tiles; t += 2 * gridDim.x) {
            for (int kc = 0; kc < p.kchunks; ++kc) {
                mbar_wait(empty0 + 8u * stage, phase ^ 1u);
                mbar_expect_tx(full0 + 8u * stage, K1_A_BYTES);
                tma_load_2d(a_base + stage * K1_A_BYTES, &map_x, full0 + 8u * stage, kc * 64, t * 64);
                if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
            }
        }
        return;
    }

    const int k = warp >> 2, w = warp & 3;
    const int tid = threadIdx.x & 127;
    const uint32_t a_base = w_base + w_bytes + k * n_stages * K1_A_BYTES;
    const uint32_t full0 = bar_base + 8u * (2 * K1_MAX_STAGES * k), empty0 = full0 + 8u * K1_MAX_STAGES;
    float *stg = staging + k * 64 * S;
    const int tq = lane & 3, tr = lane >> 2;
    const float scale = (float)(65536 - p.L);            // 2^16 - (Lp - 1)
    uint32_t stage = 0, phase = 0;
    mbar_wait(wbar, 0);
    for (int t = blockIdx.x + k * gridDim.x; t < n_tiles; t += 2 * gridDim.x) {
        float acc[NB][32];
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) acc_zero(acc[nb]);
        for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(full0 + 8u * stage, phase);
            wgmma_fence();
            const uint64_t da = make_desc(a_base + stage * K1_A_BYTES);
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
                const uint64_t db = make_desc(w_base + (kc * NPAD + nb * 64) * 128);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) wgmma_f16(acc[nb], da + 2u * kk, db + 2u * kk, (kc | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) acc_fence(acc[nb]);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + 8u * stage);
            if (++stage == (uint32_t)n_stages) { stage = 0; phase ^= 1u; }
        }
        // accumulators (+ bias, the same add as the plain kernel's epilogue) -> staging [pixel][channel]
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int row = 16 * w + tr + 8 * ((i >> 1) & 1), col = nb * 64 + 8 * (i >> 2) + 2 * tq + (i & 1);
                stg[row * S + col] = acc[nb][i] + (col < KP ? __ldg(p.bias + col) : 0.f);
            }
        wg_sync(k);
        // thread = (pixel tid % 64, channels of parity tid / 64)
        const int r = tid & 63, par = tid >> 6;
        const long long pix = (long long)t * 64 + r;
        const bool valid = pix < p.M;
        const int n = valid ? (int)(pix / p.HW) : 0;
        const int q = valid ? (int)(pix % p.HW) : 0;
        const float *row = stg + r * S;
        // the RGB coefficients condition channels 1 and 2 on the symbols of channels 0 and 1
        const float xr = (RGB && valid) ? (float)p.sym[((size_t)n * C + 0) * p.HW + q] : 0.f;
        const float xg = (RGB && valid) ? (float)p.sym[((size_t)n * C + 1) * p.HW + q] : 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            if ((c & 1) != par) continue;
            float logit[K], mean[K], logs[K], co0[K], co1[K];
#pragma unroll
            for (int kk = 0; kk < K; ++kk) {
                logit[kk] = row[0 * C * K + c * K + kk];
                mean[kk] = row[1 * C * K + c * K + kk];
                logs[kk] = row[2 * C * K + c * K + kk];
                co0[kk] = co1[kk] = 0.f;
                if (RGB && c == 1) co0[kk] = row[3 * C * K + 0 * K + kk];
                if (RGB && c == 2) {
                    co0[kk] = row[3 * C * K + 1 * K + kk];
                    co1[kk] = row[3 * C * K + 2 * K + kk];
                }
            }
            ChanParams<K> cp;
            channel_params_core<K>(logit, mean, logs, co0, co1, c, RGB, xr, xg, cp);
            const size_t so = ((size_t)n * C + c) * p.HW + q;
            const int s = valid ? (int)p.sym[so] : 0;
            const uint32_t lo = mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(p.targets + s), scale, s);
            const uint32_t hi = (s == p.L - 1) ? 0x10000u
                                               : mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(p.targets + s + 1),
                                                                    scale, s + 1);
            if (valid) p.intervals[so] = lo | ((hi - 1u) << 16);
        }
        wg_sync(k);                                      // staging is rewritten by the next tile
    }
}

}  // namespace f16

// dynamic shared memory a conv CTA may take (bytes).  Default: everything an SM has (227 KB).  L3C_CONV_SMEM_KB
// lowers it so that small latency-bound CTAs (the range decoders: 16 KB per stream) can be resident BESIDE a
// conv CTA when no SM partition separates them (codec.lanes, L3C_SM_PARTITION=0).  l3c_set_conv_launch_limits
// overrides both at the next launch.
static int conv_smem_cap() {
    static const int env_kb = [] {
        const char *e = getenv("L3C_CONV_SMEM_KB");
        return e ? atoi(e) : 227;
    }();
    const int over = conv_smem_kb_override();
    int kb = over > 0 ? over : env_kb;
    if (kb < 112) kb = 112;
    if (kb > 227) kb = 227;
    return kb * 1024;
}

namespace f16 {
template <int KIND, int NB>
static int launch_1x1(const CUtensorMap &map_x, const CUtensorMap &map_w, const Params1 &q, int n_stages,
                      int n_tiles, int grid, int smem_bytes, cudaStream_t st) {
    static bool configured_dev[64] = {};
    bool &configured = configured_dev[current_device_slot()];
    if (!configured) {
        L3C_CUDA(cudaFuncSetAttribute(conv1x1_tc_kernel<KIND, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        configured = true;
    }
    conv1x1_tc_kernel<KIND, NB><<<grid, THREADS, smem_bytes, st>>>(map_x, map_w, q, n_stages, n_tiles);
    L3C_LAUNCH_CHECK(KIND == 0 ? "conv1x1_tf32_kernel" : KIND == 1 ? "conv1x1_f16_kernel" : "conv1x1_f16x2_kernel");
    return L3C_OK;
}
}  // namespace f16

// 1x1 layers of the three tensor-core precisions.  Operand images: tf32 fp32 [M][x_pitch] (TF32-rounded), f16
// fp16 [M][x_pitch], f16x2 split fp16 [M][x_pitch = 2*Cin] (hi | lo); weight images as in conv1x1_tc_kernel.
int conv1x1_tc(const l3c_conv_t &p, cudaStream_t st) {
    using namespace f16;
    const int kind = p.precision == L3C_PREC_TF32 ? 0 : p.precision == L3C_PREC_F16 ? 1 : 2;
    L3C_REQUIRE(p.ksize == 1 && p.stride == 1 && p.Cin % 64 == 0 && p.Cin >= 64 && !(p.flags & L3C_CONV_PIXEL_SHUFFLE2) &&
                    p.x_pitch == (kind == 2 ? 2 : 1) * p.Cin,
                "l3c_conv2d: 1x1 tensor-core layers need Cin %% 64 == 0 and a dense input pitch (got Cin=%d pitch=%d)",
                p.Cin, p.x_pitch);
    L3C_REQUIRE(p.cout_pad % 64 == 0 && p.cout_pad >= p.Cout && p.cout_pad <= 256,
                "l3c_conv2d: 1x1 tensor-core layers are built for Cout <= 256 (got %d, cout_pad=%d)", p.Cout, p.cout_pad);
    if (kind == 0) {
        L3C_REQUIRE(p.x && p.w && p.y, "l3c_conv2d[tf32]: x / w / y are required");
    } else {
        L3C_REQUIRE(p.Cout % 2 == 0 && p.y_pitch % 2 == 0 && p.y_coff % 2 == 0,
                    "l3c_conv2d: 1x1 layers need even Cout/pitch/offset");
        L3C_REQUIRE(!p.residual, "l3c_conv2d: residual on a 1x1 layer is not built");
        L3C_REQUIRE(p.x_h && p.w_h, "l3c_conv2d: x_h / w_h (fp16 operand images) are required");
        L3C_REQUIRE(kind == 1 ? (p.y || p.y_h) : (p.y && !p.y_h), "l3c_conv2d: 1x1 layer outputs (f16: fp32 and / or "
                                                                  "FP16 image; f16x2: fp32 only)");
    }
    EncodeTiledFn encode = get_encode_fn();
    L3C_REQUIRE(encode != nullptr, "l3c_conv2d: cuTensorMapEncodeTiled is not available from the driver");
    const int planes = kind == 2 ? 2 : 1;
    const int kunits = kind == 0 ? p.Cin / 32 : p.Cin / 64;
    const long long M = (long long)p.N * p.H * p.W;
    const int w_plane = kunits * p.cout_pad * 128;
    const int sb = planes * K1_A_BYTES;
    const int cap = kind == 1 ? conv_smem_cap() : 227 * 1024;
    int n_stages = (cap - 1024 - 512 - planes * w_plane) / (2 * sb);
    if (n_stages < 1 && planes * w_plane + 2 * sb <= 227 * 1024 - 1024 - 512) n_stages = 1;   // above the cap
    if (n_stages > K1_MAX_STAGES) n_stages = K1_MAX_STAGES;
    L3C_REQUIRE(n_stages >= 1, "l3c_conv2d: weights of a %d -> %d 1x1 layer do not fit in shared memory", p.Cin, p.Cout);
    const CUtensorMapDataType dt = kind == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const int esz = kind == 0 ? 4 : 2, ch = kind == 0 ? 32 : 64;
    alignas(64) CUtensorMap map_x, map_w;
    {
        cuuint64_t dims[2] = {(cuuint64_t)p.x_pitch, (cuuint64_t)M};
        cuuint64_t strides[1] = {(cuuint64_t)p.x_pitch * esz};
        cuuint32_t box[2] = {(cuuint32_t)ch, 64};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&map_x, dt, 2, const_cast<void *>(kind == 0 ? (const void *)p.x : p.x_h), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d: cuTensorMapEncodeTiled(x, 1x1) failed with %d", (int)r);
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)ch, (cuuint64_t)planes * kunits * p.cout_pad};
        cuuint64_t strides[1] = {128};
        cuuint32_t box[2] = {(cuuint32_t)ch, (cuuint32_t)p.cout_pad};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&map_w, dt, 2, const_cast<void *>(kind == 0 ? (const void *)p.w : p.w_h), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d: cuTensorMapEncodeTiled(w, 1x1) failed with %d", (int)r);
    }
    const int nblk = p.cout_pad / 64;
    const int nb = kind == 2 ? (nblk % 2 == 0 ? 2 : 1) : nblk;     // f16x2: two accumulators per block
    Params1 q;
    q.bias = p.bias; q.residual = p.residual; q.y = p.y; q.y_tf32 = p.y_tf32;
    q.yh = reinterpret_cast<__half *>(p.y_h);
    q.M = M; q.Cout = p.Cout; q.y_pitch = p.y_pitch; q.y_coff = p.y_coff; q.flags = p.flags;
    q.kunits = kunits; q.npad = p.cout_pad; q.lo_ch = p.Cin; q.nch = nblk / nb;
    const long long n_tiles64 = (M + 63) / 64 * q.nch;
    L3C_REQUIRE(n_tiles64 < (1ll << 31), "l3c_conv2d: 1x1 layer too large (%lld pixels)", M);
    const int n_tiles = (int)n_tiles64;
    const int n_sm = stream_sm_count(st);
    const int grid = ceil_div(n_tiles, 2) < n_sm ? ceil_div(n_tiles, 2) : n_sm;
    const int smem_bytes = planes * w_plane + 2 * n_stages * sb + 1024 + 512;
#define L3C_1X1(K_, NB_) \
    if (kind == K_ && nb == NB_) return launch_1x1<K_, NB_>(map_x, map_w, q, n_stages, n_tiles, grid, smem_bytes, st)
    L3C_1X1(0, 1); L3C_1X1(0, 2); L3C_1X1(0, 3); L3C_1X1(0, 4);
    L3C_1X1(1, 1); L3C_1X1(1, 2); L3C_1X1(1, 3); L3C_1X1(1, 4);
    L3C_1X1(2, 1); L3C_1X1(2, 2);
#undef L3C_1X1
    set_error("l3c_conv2d: no 1x1 kernel for precision %d, %d channel blocks", p.precision, nb);
    return L3C_EINVAL;
}

// operand image x_h: fp16 NHWC [N][H][W][x_pitch]; weight image w_h (engine.PackedConv.get_f16):
//   3x3: [tap 9][cout_pad][64] fp16      5x5: [tap 25][cout_pad][64]      1x1: [Cin/64][cout_pad][64] (rows of 128 B)
int conv2d_f16(const l3c_conv_t &p, cudaStream_t st) {
    using namespace f16;
    const bool k3 = p.ksize == 3 && p.stride == 1 && p.Cin == 64 && p.x_pitch == 64;
    const bool k5 = p.ksize == 5 && p.stride == 2 && p.dilation == 1 && p.Cin == 64 && p.x_pitch == 64;
    const bool k1 = p.ksize == 1 && p.stride == 1 && p.Cin % 64 == 0 && p.x_pitch == p.Cin &&
                    !(p.flags & L3C_CONV_PIXEL_SHUFFLE2);
    L3C_REQUIRE(k3 || k5 || k1, "l3c_conv2d[f16]: tensor-core path needs 3x3/s1/Cin=64, 5x5/s2/Cin=64 or 1x1/Cin%%64==0, "
                                "dense input pitch (got k=%d s=%d Cin=%d pitch=%d)", p.ksize, p.stride, p.Cin, p.x_pitch);
    L3C_REQUIRE(p.x_h && p.w_h, "l3c_conv2d[f16]: x_h / w_h (fp16 operand images) are required");
    L3C_REQUIRE(p.y || p.y_h, "l3c_conv2d[f16]: no output");
    L3C_REQUIRE(p.cout_pad % 64 == 0 && p.cout_pad >= p.Cout, "l3c_conv2d[f16]: cout_pad=%d", p.cout_pad);
    L3C_REQUIRE(!(p.flags & ~(L3C_CONV_RELU | L3C_CONV_PIXEL_SHUFFLE2)), "l3c_conv2d[f16]: unsupported flags %u", p.flags);
    if (k1) return conv1x1_tc(p, st);
    EncodeTiledFn encode = get_encode_fn();
    L3C_REQUIRE(encode != nullptr, "l3c_conv2d: cuTensorMapEncodeTiled is not available from the driver");
    const int n_sm = stream_sm_count(st);          // the stream may be confined to a group of SMs
    static bool configured_dev[64] = {};
    bool &configured = configured_dev[current_device_slot()];
    if (!configured) {
        L3C_CUDA(cudaFuncSetAttribute(conv_f16_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        L3C_CUDA(cudaFuncSetAttribute(conv_f16_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        configured = true;
    }
    alignas(64) CUtensorMap map_x, map_w;
    if (k3) {
        L3C_REQUIRE(p.Cout % 64 == 0, "l3c_conv2d[f16]: 3x3 layers need Cout %% 64 == 0 (got %d)", p.Cout);
        const bool ps = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
        L3C_REQUIRE(ps ? (p.y_pitch % 2 == 0 && p.y_coff % 2 == 0) : (p.y_pitch % 8 == 0 && p.y_coff % 8 == 0),
                    "l3c_conv2d[f16]: output pitch/offset alignment (pitch=%d coff=%d)", p.y_pitch, p.y_coff);
        L3C_REQUIRE(!(ps && p.residual), "l3c_conv2d[f16]: residual with pixel shuffle is not built");
        const int d = p.dilation;
        const int a_rows = TH + 2 * d;
        L3C_REQUIRE(a_rows <= 256, "l3c_conv2d[f16]: dilation %d too large", d);
        const int a_bytes = a_rows * TW * 128;
        int n_stages = (conv_smem_cap() - 1024 - 512 - W_RES_BYTES) / (2 * a_bytes);      // per pipe
        if (n_stages > 3) n_stages = 3;
        if (n_stages < 1 && 2 * a_bytes <= 227 * 1024 - 1024 - 512 - W_RES_BYTES) n_stages = 1;   // above the cap
        L3C_REQUIRE(n_stages >= 1, "l3c_conv2d[f16]: halo of dilation %d does not fit in shared memory", d);
        {
            cuuint64_t dims[4] = {64, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
            cuuint64_t strides[3] = {128, (cuuint64_t)p.W * 128, (cuuint64_t)p.H * p.W * 128};
            cuuint32_t box[4] = {64, TW, (cuuint32_t)a_rows, 1};
            cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = encode(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(p.x_h), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d[f16]: cuTensorMapEncodeTiled(x) failed with %d", (int)r);
        }
        {
            cuuint64_t dims[2] = {64, (cuuint64_t)9 * p.cout_pad};
            cuuint64_t strides[1] = {128};
            cuuint32_t box[2] = {64, 64};
            cuuint32_t estr[2] = {1, 1};
            CUresult r = encode(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(p.w_h), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d[f16]: cuTensorMapEncodeTiled(w) failed with %d", (int)r);
        }
        Params q;
        q.bias = p.bias; q.residual = p.residual; q.y = p.y; q.yh = reinterpret_cast<__half *>(p.y_h);
        q.N = p.N; q.H = p.H; q.W = p.W;
        q.Cout = p.Cout; q.y_pitch = p.y_pitch; q.y_coff = p.y_coff;
        q.dilation = d; q.flags = p.flags;
        q.tiles_x = ceil_div(p.W, TW);
        q.tiles_y = ceil_div(p.H, TH);
        const int cout_tiles = p.cout_pad / 64;
        const int ptiles = p.N * q.tiles_x * q.tiles_y;
        int per_ct = n_sm / cout_tiles;
        if (per_ct < 1) per_ct = 1;
        if (per_ct > ptiles) per_ct = ptiles;
        const int smem_bytes = W_RES_BYTES + 2 * n_stages * a_bytes + 1024 + 512;
        conv_f16_kernel<0><<<dim3(per_ct, cout_tiles), THREADS, smem_bytes, st>>>(map_x, map_w, q, n_stages, a_bytes, ptiles);
        L3C_LAUNCH_CHECK("conv3x3_f16_kernel");
        return L3C_OK;
    }
    // ---- 5x5 / stride 2
    L3C_REQUIRE(p.Cout % 64 == 0, "l3c_conv2d[f16]: 5x5/s2 layers need Cout %% 64 == 0 (got %d)", p.Cout);
    L3C_REQUIRE(!(p.flags & L3C_CONV_PIXEL_SHUFFLE2) && p.y_pitch % 8 == 0 && p.y_coff % 8 == 0,
                "l3c_conv2d[f16]: 5x5/s2 output pitch/offset alignment (pitch=%d coff=%d)", p.y_pitch, p.y_coff);
    const int Ho = (p.H + 4 - 5) / 2 + 1, Wo = (p.W + 4 - 5) / 2 + 1;
    {
        // element strides (2, 2): the box visits every second pixel / row; box sizes are given in
        // traversed elements (16 px -> 32, 10 rows -> 20)
        cuuint64_t dims[4] = {64, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
        cuuint64_t strides[3] = {128, (cuuint64_t)p.W * 128, (cuuint64_t)p.H * p.W * 128};
        cuuint32_t box[4] = {64, 2 * TW, 20, 1};
        cuuint32_t estr[4] = {1, 2, 2, 1};
        CUresult r = encode(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(p.x_h), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d[f16]: cuTensorMapEncodeTiled(x, 5x5/s2) failed with %d", (int)r);
    }
    {
        cuuint64_t dims[2] = {64, (cuuint64_t)25 * p.cout_pad};
        cuuint64_t strides[1] = {128};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(p.w_h), dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_conv2d[f16]: cuTensorMapEncodeTiled(w, 5x5/s2) failed with %d", (int)r);
    }
    Params q;
    q.bias = p.bias; q.residual = p.residual; q.y = p.y; q.yh = reinterpret_cast<__half *>(p.y_h);
    q.N = p.N; q.H = Ho; q.W = Wo;                      // the epilogue works on OUTPUT pixels
    q.Cout = p.Cout; q.y_pitch = p.y_pitch; q.y_coff = p.y_coff;
    q.dilation = 1; q.flags = p.flags;
    q.tiles_x = ceil_div(Wo, TW);
    q.tiles_y = ceil_div(Ho, TH);
    const int cout_tiles = p.cout_pad / 64;
    const int ptiles = p.N * q.tiles_x * q.tiles_y;
    int per_ct = n_sm / cout_tiles;
    if (per_ct < 1) per_ct = 1;
    if (per_ct > ptiles) per_ct = ptiles;
    const int n_stages = (conv_smem_cap() - 1024 - 512) / (2 * K5_STAGE_BYTES) >= 2 ? 2 : 1;
    const int smem_bytes = 2 * n_stages * K5_STAGE_BYTES + 1024 + 512;
    conv_f16_kernel<1><<<dim3(per_ct, cout_tiles), THREADS, smem_bytes, st>>>(map_x, map_w, q, n_stages, K5_STAGE_BYTES, ptiles);
    L3C_LAUNCH_CHECK("conv5x5s2_f16_kernel");
    return L3C_OK;
}

}  // namespace l3c

// 1x1 conv (Cin % 64 == 0 -> Kp = (rgb ? 4 : 3) * C * 10 parameters) fused with the per-symbol coding intervals
extern "C" int l3c_lin_dmll_intervals(const void *x_h, const void *w_h, const float *bias, const uint8_t *sym_dev,
                                      const float *targets_dev, int N, int HW, int Cin, int C, int K, int L, int rgb,
                                      uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    using namespace l3c::f16;
    L3C_REQUIRE(x_h && w_h && bias && sym_dev && targets_dev && intervals_dev, "l3c_lin_dmll_intervals: null pointer");
    L3C_REQUIRE(N >= 1 && HW >= 1 && Cin % 64 == 0 && Cin >= 64, "l3c_lin_dmll_intervals: N=%d HW=%d Cin=%d", N, HW, Cin);
    L3C_REQUIRE(K == 10 && L >= 2 && L <= 256, "l3c_lin_dmll_intervals: K=%d L=%d (only K=10 is built)", K, L);
    L3C_REQUIRE((rgb && C == 3) || (!rgb && C == 5), "l3c_lin_dmll_intervals: built for RGB (C=3) and C=5 bottlenecks, "
                                                     "got C=%d rgb=%d", C, rgb);
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int npad = (Kp + 63) / 64 * 64;            // 128 (RGB) / 192
    cudaStream_t st = (cudaStream_t)stream;
    EncodeTiledFn encode = get_encode_fn();
    L3C_REQUIRE(encode != nullptr, "l3c_lin_dmll_intervals: cuTensorMapEncodeTiled is not available from the driver");
    static bool configured_dev[64] = {};
    bool &configured = configured_dev[current_device_slot()];
    if (!configured) {
        L3C_CUDA(cudaFuncSetAttribute(lin_dmll_f16_kernel<3, true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        L3C_CUDA(cudaFuncSetAttribute(lin_dmll_f16_kernel<5, false, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        configured = true;
    }
    const int kchunks = Cin / 64;
    const long long M = (long long)N * HW;
    const int w_bytes = kchunks * npad * 128;
    const int stg_bytes = 2 * 64 * (npad + 1) * 4 + 64;
    int n_stages = (conv_smem_cap() - 1024 - 512 - w_bytes - stg_bytes) / (2 * K1_A_BYTES);
    if (n_stages < 1 && w_bytes + stg_bytes + 2 * K1_A_BYTES <= 227 * 1024 - 1024 - 512) n_stages = 1;
    if (n_stages > K1_MAX_STAGES) n_stages = K1_MAX_STAGES;
    L3C_REQUIRE(n_stages >= 1, "l3c_lin_dmll_intervals: weights do not fit in shared memory (Cin=%d)", Cin);
    alignas(64) CUtensorMap map_x, map_w;
    {
        cuuint64_t dims[2] = {(cuuint64_t)Cin, (cuuint64_t)M};
        cuuint64_t strides[1] = {(cuuint64_t)Cin * 2};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(x_h), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_lin_dmll_intervals: cuTensorMapEncodeTiled(x) failed with %d", (int)r);
    }
    {
        cuuint64_t dims[2] = {64, (cuuint64_t)kchunks * npad};
        cuuint64_t strides[1] = {128};
        cuuint32_t box[2] = {64, (cuuint32_t)npad};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(w_h), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        L3C_REQUIRE(r == CUDA_SUCCESS, "l3c_lin_dmll_intervals: cuTensorMapEncodeTiled(w) failed with %d", (int)r);
    }
    ParamsLD q;
    q.bias = bias; q.sym = sym_dev; q.targets = targets_dev; q.intervals = intervals_dev;
    q.M = M; q.HW = HW; q.L = L; q.kchunks = kchunks; q.npad = npad;
    const int n_tiles = (int)((M + 63) / 64);
    const int n_sm = stream_sm_count(st);
    const int grid = ceil_div(n_tiles, 2) < n_sm ? ceil_div(n_tiles, 2) : n_sm;
    const int smem_bytes = w_bytes + 2 * n_stages * K1_A_BYTES + stg_bytes + 1024 + 512;
    if (rgb)
        lin_dmll_f16_kernel<3, true, 2><<<grid, THREADS, smem_bytes, st>>>(map_x, map_w, q, n_stages, n_tiles);
    else
        lin_dmll_f16_kernel<5, false, 3><<<grid, THREADS, smem_bytes, st>>>(map_x, map_w, q, n_stages, n_tiles);
    L3C_LAUNCH_CHECK("lin_dmll_f16_kernel");
    return L3C_OK;
}
