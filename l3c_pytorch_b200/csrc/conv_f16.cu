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
//     box is one TMA load (no K-halves) and half the L2->smem bytes;
//   * operand twins cost 128 instead of 256 B per pixel in HBM, and a layer whose output only feeds tensor-core
//     convs (first conv of a ResBlock, atrous convs, the finest decoder features) writes ONLY the 2-byte image.
// Per pixel a 64->64 conv moves 256 B (operand in / operand out) to 768 B (operand + fp32 residual in, fp32 +
// operand out) against 73.7 kFLOP.
//
// Structure of the 3x3 kernel (persistent, tc_conv.cuh layout: two consumer warpgroups with a TMA producer warp
// each):
//   * the 9 weight slabs of the CTA's Cout tile (9 x 64 rows x 128 B = 72 KB) stay in shared memory;
//   * per tile ONE halo box of (8 + 2d) rows x halo_w(d) pixels (24 for d <= 4) x 64 channels is staged by TMA,
//     so every input pixel crosses L2 -> smem once per tile (240 / 288 / 384 B per output pixel at d = 1 / 2 / 4
//     instead of three boxes of 16 px, one per filter column, at twice that);
//   * the two 64-pixel halves of the 8x16 tile are its left and right 8-pixel columns (Halves::COLS): the 8-row
//     core-matrix groups of a half are 8 box rows one box row (a multiple of 1024 B) apart, so every tap (dy, dx)
//     of a half is one descriptor, started at pixel dx*d, i.e. anywhere inside the swizzle atom (halo_mma);
//   * the consumer warpgroup accumulates both halves (2 x 32 registers per thread), then fuses bias / ReLU /
//     residual / PixelShuffle(2), writes fp32 float2 (full sectors) and the FP16 image as 16-byte vectors after a
//     4x4 transpose inside each quad.
// Accumulation order per output element: (dx, dy, k-step) -- fixed, independent of batch / image size / tile
// position / pipe: encoder-side and decoder-side evaluations are bit-identical.
#include <stdlib.h>

#include "tc_conv.cuh"
#include "dmll_math.cuh"

namespace l3c {
namespace f16 {
using namespace tcx;

constexpr int W_TAP_BYTES = 64 * 128;          // one filter tap of one Cout tile: 64 rows x 64 fp16
constexpr int W_RES_BYTES = 9 * W_TAP_BYTES;   // 73728

// KIND 0: 3x3 stride 1 (any dilation), weights resident.
// KIND 1: 5x5 stride 2 (the down-sampling conv of every encoder, net.py:101): the input box of a tap is read
//   with TMA element strides (2, 2), so the A operand of an 8x16 OUTPUT tile is again 128 dense rows of 128 B;
//   for a filter column kx the taps ky = 0,2,4 (and ky = 1,3) share one strided box of 10 rows read at row
//   offsets j*2048 B.  25 taps x 8 KB of weights do not fit beside the stages: every unit (kx, row parity)
//   brings its 3 (2) weight slabs along with its box.  10 units, 100 k-steps per tile.
constexpr int K5_A_BYTES = 10 * TW * 128;                  // 20480: strided halo box
constexpr int K5_STAGE_BYTES = K5_A_BYTES + 3 * W_TAP_BYTES;   // 45056: box + up to three weight slabs

// KIND 0: width (pixels) of the halo box, TW + 2d rounded up to whole 8-pixel groups so that one box row (the
// descriptors' SBO) is a multiple of the 1024 B swizzle atom.  24 for d = 1..4.
__host__ __device__ constexpr int halo_w(int d) { return (TW + 2 * d + 7) & ~7; }

// The 72 wgmmas of a 3x3 tile on its halo box (bw pixels wide, its row 0 / pixel 0 the input row / pixel d before
// the tile's first): tap (dy, dx) of half h reads box rows dy*d + g (g = 0..7, the tile rows), pixels
// 8h + dx*d + 0..7.  Every output element accumulates in the order (dx, dy, k-step); the two halves alternate
// per k-step, which measured ~1 % faster than four k-steps of one half after the other.
__device__ __forceinline__ void halo_mma(float (&acc)[2][32], uint32_t box, int d, int bw, uint32_t w_base) {
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const uint64_t db = make_desc(w_base + (dy * 3 + dx) * W_TAP_BYTES);
            const uint32_t a0 = box + (dy * d * bw + dx * d) * 128;
            const uint64_t da[2] = {make_desc(a0, bw * 128), make_desc(a0 + 8 * 128, bw * 128)};
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)                                          // +32 B = 16 fp16 along K
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    wgmma_f16(acc[h], da[h] + 2u * kk, db + 2u * kk, (dx | dy | kk) != 0 ? 1u : 0u);
        }
    }
}

// The wgmmas of one unit of an 8x16 tile: NTAPS taps j, tap j reading the staged box at a0 from row j * row_step
// (rows of 16 pixels) and the weight slab at w0 + j * w_step, each for both 64-pixel halves and four k-steps.
// `first`: the unit starts the tile's accumulation (its first k-step overwrites the accumulators).
template <int NTAPS>
__device__ __forceinline__ void unit_mma(float (&acc)[2][32], uint32_t a0, int row_step, uint32_t w0, uint32_t w_step,
                                         bool first) {
#pragma unroll
    for (int j = 0; j < NTAPS; ++j) {
        const uint64_t db = make_desc(w0 + j * w_step);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint64_t da = make_desc(a0 + (j * row_step * TW + 64 * h) * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)                                          // +32 B = 16 fp16 along K
                wgmma_f16(acc[h], da + 2u * kk, db + 2u * kk, (first && j == 0 && kk == 0) ? 0u : 1u);
        }
    }
}

template <int KIND>
__global__ void __launch_bounds__(THREADS, 1)
conv_f16_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                const Params p, const int n_stages, const int a_bytes, const int ptiles,
                const TileSchedule ts) {
    L3C_TRACE_BEGIN;
    constexpr int W_RES = (KIND == 0) ? W_RES_BYTES : 0;    // resident weights
    constexpr int UNITS = (KIND == 0) ? 1 : 10;
    constexpr Halves HV = (KIND == 0) ? Halves::COLS : Halves::ROWS;
    // [weights 72 KB][pipe 0 stages][pipe 1 stages][barriers]
    const uint32_t w_base = smem_u32(smem_aligned());
    const uint32_t bars = w_base + W_RES + 2 * n_stages * a_bytes;
    pipeline_init(bars, &map_x, &map_w);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k = warp < CONSUMER_WARPS ? warp >> 2 : warp - CONSUMER_WARPS;   // pipe
    const int d = p.dilation;
    const int ct = blockIdx.y;                        // this CTA's Cout tile (weights stay resident)
    Ring ring(w_base + W_RES, a_bytes, n_stages, bars, k);
    TileQueue tiles(bars, k, 2, ptiles, ts);

    if (warp >= CONSUMER_WARPS) {
        // ===================== TMA producer of pipe k =====================
        if (lane != 0) return;
        if (KIND == 0 && k == 0) {
            mbar_expect_tx(weight_bar(bars), W_RES_BYTES);
            for (int tap = 0; tap < 9; ++tap)         // rows [tap][cout_pad] of the weight image
                tma_load_2d(w_base + tap * W_TAP_BYTES, &map_w, weight_bar(bars), 0, tap * (int)gridDim.y * 64 + ct * 64);
        }
        produce_tiles(tiles, [&](int t) {
            const Tile c = tile_of(p, t);
            for (int u = 0; u < UNITS; ++u) {
                if (KIND == 0) {
                    const Slot s = ring.acquire(a_bytes);       // the tile's halo box
                    tma_load_4d(s.dst, &map_x, s.bar, 0, c.tx * TW - d, c.ty * TH - d, c.n);
                } else {
                    const int kx = u >> 1, par = u & 1, ntaps = 3 - par;
                    const Slot s = ring.acquire(K5_A_BYTES + ntaps * W_TAP_BYTES);
                    // input pixel of output (oy, ox), tap (ky, kx): (2*oy + ky - 2, 2*ox + kx - 2)
                    tma_load_4d(s.dst, &map_x, s.bar, 0, 2 * c.tx * TW + kx - 2, 2 * c.ty * TH + par - 2, c.n);
                    for (int j = 0; j < ntaps; ++j)
                        tma_load_2d(s.dst + K5_A_BYTES + j * W_TAP_BYTES, &map_w, s.bar, 0,
                                    ((par + 2 * j) * 5 + kx) * (int)gridDim.y * 64 + ct * 64);
                }
            }
        });
        return;
    }

    // ===================== consumer warpgroup k: wgmma + epilogue =====================
    const int w = warp & 3;
    if (KIND == 0) mbar_wait(weight_bar(bars), 0);
    consume_tiles(tiles, [&](int t) {
        const Tile c = tile_of(p, t);
        prefetch_residual<HV>(p, c, ct, w);
        float acc[2][32];                                 // the two halves of the tile (HV)
        acc_zero(acc[0]);
        acc_zero(acc[1]);
        // one unit: wait for its stage, issue(stage address) its wgmmas as one group, wait for them, hand it back
        auto unit = [&](auto &&issue) {
            const uint32_t a0 = ring.wait();
            wgmma_fence();
            issue(a0);
            wgmma_commit();
            wgmma_wait0();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            ring.release();
        };
        if (KIND == 0) {
            const int bw = halo_w(d);
            unit([&](uint32_t a0) { halo_mma(acc, a0, d, bw, w_base); });   // all 9 taps on the one halo box
        } else {
            // unit (kx, row parity): taps ky = par + 2j, box row j, weight slab j after the box.  The two parities
            // are separate bodies so that both tap loops have compile-time trip counts: with a runtime count ptxas
            // serialises every wgmma of the kernel.
            for (int kx = 0; kx < 5; ++kx) {
                unit([&](uint32_t a0) { unit_mma<3>(acc, a0, 1, a0 + K5_A_BYTES, W_TAP_BYTES, kx == 0); });
                unit([&](uint32_t a0) { unit_mma<2>(acc, a0, 1, a0 + K5_A_BYTES, W_TAP_BYTES, false); });
            }
        }
        image_epilogue<false, HV>(p, c, ct, w, acc);
    });
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

// Producer of a 1x1 pipe: pipe 0 first loads the resident weights (PLANES x kunits K chunks of npad rows), then
// each tile t (pixel tile t / nch) stages its kunits K chunks of 64 pixels, in KIND 2 with their lo plane.
// tpi > 0 (a band, lin_dmll_f16_kernel): map_x is 3-D [N][pixels][channels] and pixel tile pt is tile pt % tpi of
// image pt / tpi.
template <int KIND, bool BAND = false>
__device__ __forceinline__ void produce_1x1(Ring &ring, const CUtensorMap *map_x, const CUtensorMap *map_w,
                                            TileQueue &tiles, uint32_t w_base, uint32_t wbar, int k, int kunits,
                                            int npad, int nch, int lo_ch, int tpi = 0) {
    constexpr int PLANES = (KIND == 2) ? 2 : 1;
    constexpr int CH = (KIND == 0) ? 32 : 64;           // channels per K chunk
    if (k == 0) {
        mbar_expect_tx(wbar, (uint32_t)(PLANES * kunits * npad * 128));
        for (int kc = 0; kc < PLANES * kunits; ++kc)
            tma_load_2d(w_base + kc * npad * 128, map_w, wbar, 0, kc * npad);
    }
    produce_tiles(tiles, [&](int t) {
        const int pt = t / nch;
        for (int u = 0; u < kunits; ++u) {
            const Slot s = ring.acquire(PLANES * K1_A_BYTES);
            if constexpr (BAND) {
                tma_load_3d(s.dst, map_x, s.bar, u * CH, (pt % tpi) * 64, pt / tpi);
            } else {
                tma_load_2d(s.dst, map_x, s.bar, u * CH, pt * 64);
                if (KIND == 2) tma_load_2d(s.dst + K1_A_BYTES, map_x, s.bar, lo_ch + u * CH, pt * 64);
            }
        }
    });
}

// Mainloop of a 1x1 tile: acc[nb] (KIND 2: acc1 = acc, acc2) over all K chunks for the output channels
// (nc * NB + nb) * 64 + 0..63; the lo weight plane starts w_plane bytes after the hi plane.
template <int KIND, int NB>
__device__ __forceinline__ void mma_1x1(Ring &ring, float (&acc)[NB][32], float (&acc2)[NB][32], uint32_t w_base,
                                        int w_plane, int kunits, int npad, int nc) {
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) acc_zero(acc[nb]);
    if (KIND == 2) {
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) acc_zero(acc2[nb]);
    }
    for (int u = 0; u < kunits; ++u) {
        const uint32_t a0 = ring.wait();
        wgmma_fence();
        const uint64_t ah = make_desc(a0);
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
            const int col = (nc * NB + nb) * 64;
            const uint64_t bh = make_desc(w_base + (u * npad + col) * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t first = (u | kk) != 0 ? 1u : 0u;
                if (KIND == 0) {
                    wgmma_tf32(acc[nb], ah + 2u * kk, bh + 2u * kk, first);
                } else {
                    wgmma_f16(acc[nb], ah + 2u * kk, bh + 2u * kk, first);
                    if (KIND == 2) {
                        const uint64_t al = make_desc(a0 + K1_A_BYTES);
                        const uint64_t bl = make_desc(w_base + w_plane + (u * npad + col) * 128);
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
        ring.release();
    }
}

template <int KIND, int NB>
__global__ void __launch_bounds__(THREADS, 1)
conv1x1_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                  const Params1 p, const int n_stages, const int n_tiles, const TileSchedule ts) {
    L3C_TRACE_BEGIN;
    constexpr int PLANES = (KIND == 2) ? 2 : 1;
    const int w_plane = p.kunits * p.npad * 128;
    // [weights (hi plane, lo plane)][pipe 0 stages][pipe 1 stages][barriers]
    const uint32_t w_base = smem_u32(smem_aligned());
    const uint32_t bars = w_base + PLANES * w_plane + 2 * n_stages * PLANES * K1_A_BYTES;
    pipeline_init(bars, &map_x, &map_w);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k = warp < CONSUMER_WARPS ? warp >> 2 : warp - CONSUMER_WARPS;   // pipe
    Ring ring(w_base + PLANES * w_plane, PLANES * K1_A_BYTES, n_stages, bars, k);
    TileQueue tiles(bars, k, 2, n_tiles, ts);

    if (warp >= CONSUMER_WARPS) {
        if (lane == 0)
            produce_1x1<KIND>(ring, &map_x, &map_w, tiles, w_base, weight_bar(bars), k, p.kunits, p.npad, p.nch, p.lo_ch);
        return;
    }

    // ===================== consumer warpgroup k =====================
    const int w = warp & 3;
    const int tq = lane & 3, tr = lane >> 2;
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool round_y = (p.flags & L3C_CONV_ROUND_TF32) != 0;
    mbar_wait(weight_bar(bars), 0);
    consume_tiles(tiles, [&](int t) {
        const int pt = t / p.nch, nc = t % p.nch;
        float acc[NB][32], acc2[NB][32];          // acc2: KIND 2 only
        mma_1x1<KIND, NB>(ring, acc, acc2, w_base, w_plane, p.kunits, p.npad, nc);
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
    });
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
    static constexpr bool BAND = false;
};

// A band of a banded encode (l3c_lin_dmll_intervals_band): x is the band's rows of a window's concat buffer, a 3-D
// TMA map [N][g.h * g.W][Cin] with the window's image stride, tpi pixel tiles per image (HW = 64 tpi, M = N HW: the
// tile numbering); sym is the whole symbol plane and the intervals go to band stream planes in tile order (BandGeom).
struct ParamsLDBand : ParamsLD {
    BandGeom g;
    int tpi;
    static constexpr bool BAND = true;
};

// A band's element of the symbol of channel c of pixel q of image n (its row of the whole symbol plane), and of its
// interval (its tile-order position in the band stream planes); the whole-plane kernel uses element (n C + c) HW + q
// for both.  The ParamsLD overloads are never called.
template <int C>
__device__ __forceinline__ size_t sym_elem(const ParamsLD &, int, int, int) { return 0; }
template <int C>
__device__ __forceinline__ size_t iv_elem(const ParamsLD &, int, int, int) { return 0; }
template <int C>
__device__ __forceinline__ size_t sym_elem(const ParamsLDBand &p, int n, int c, int q) {
    const int y = q / p.g.W;
    return ((size_t)n * C + c) * p.g.sym_hw + (long long)(p.g.y0 + y) * p.g.W + (q - y * p.g.W);
}
template <int C>
__device__ __forceinline__ size_t iv_elem(const ParamsLDBand &p, int n, int c, int q) {
    const int y = q / p.g.W;
    return ((size_t)n * C + c) * ((size_t)p.g.h * p.g.W) +
           raster_to_tile_order(y, q - y * p.g.W, p.g.h, p.g.W, p.g.th, p.g.tw);
}
// a band's images are tpi * 64 pixels apart in the tile numbering (p.HW), of which the first h * W are the band's
__device__ __forceinline__ bool in_band(const ParamsLD &, long long) { return true; }
__device__ __forceinline__ bool in_band(const ParamsLDBand &p, long long pix) {
    return pix % p.HW < (long long)p.g.h * p.g.W;
}

template <int C, bool RGB, int NB, class P = ParamsLD>
__global__ void __launch_bounds__(THREADS, 1)
lin_dmll_f16_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const P p, const int n_stages, const int n_tiles, const TileSchedule ts) {
    L3C_TRACE_BEGIN;
    constexpr int K = 10;
    constexpr int KP = (RGB ? 4 : 3) * C * K;            // parameters per pixel (the bias has KP entries)
    constexpr int NPAD = NB * 64, S = NPAD + 1;         // staging row pitch (floats): conflict-free column reads
    uint8_t *smem = smem_aligned();
    const int w_bytes = p.kchunks * NPAD * 128;
    // [weights][pipe 0 stages][pipe 1 stages][staging 2 x 64 x S fp32][barriers]
    float *staging = reinterpret_cast<float *>(smem + w_bytes + 2 * n_stages * K1_A_BYTES);
    const uint32_t w_base = smem_u32(smem);
    const uint32_t bars = smem_u32(staging + 2 * 64 * S);
    pipeline_init(bars, &map_x, &map_w);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k = warp < CONSUMER_WARPS ? warp >> 2 : warp - CONSUMER_WARPS;   // pipe
    Ring ring(w_base + w_bytes, K1_A_BYTES, n_stages, bars, k);
    TileQueue tiles(bars, k, 2, n_tiles, ts);

    if (warp >= CONSUMER_WARPS) {
        if constexpr (P::BAND) {
            if (lane == 0)
                produce_1x1<1, true>(ring, &map_x, &map_w, tiles, w_base, weight_bar(bars), k, p.kchunks, NPAD, 1, 0,
                                     p.tpi);
        } else {
            if (lane == 0) produce_1x1<1>(ring, &map_x, &map_w, tiles, w_base, weight_bar(bars), k, p.kchunks, NPAD, 1, 0);
        }
        return;
    }

    const int w = warp & 3;
    const int tid = threadIdx.x & 127;
    float *stg = staging + k * 64 * S;
    const int tq = lane & 3, tr = lane >> 2;
    const float scale = (float)(65536 - p.L);            // 2^16 - (Lp - 1)
    mbar_wait(weight_bar(bars), 0);
    consume_tiles(tiles, [&](int t) {
        float acc[NB][32];
        mma_1x1<1, NB>(ring, acc, acc, w_base, 0, p.kchunks, NPAD, 0);     // acc2 is not used by KIND 1
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
        const bool valid = pix < p.M && in_band(p, pix);
        const int n = valid ? (int)(pix / p.HW) : 0;
        const int q = valid ? (int)(pix % p.HW) : 0;
        const float *row = stg + r * S;
        // the RGB coefficients condition channels 1 and 2 on the symbols of channels 0 and 1
        const float xr = (RGB && valid) ? (float)p.sym[P::BAND ? sym_elem<C>(p, n, 0, q) : ((size_t)n * C + 0) * p.HW + q] : 0.f;
        const float xg = (RGB && valid) ? (float)p.sym[P::BAND ? sym_elem<C>(p, n, 1, q) : ((size_t)n * C + 1) * p.HW + q] : 0.f;
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
            const size_t so = P::BAND ? sym_elem<C>(p, n, c, q) : ((size_t)n * C + c) * p.HW + q;
            const int s = valid ? (int)p.sym[so] : 0;
            const uint32_t lo = mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(p.targets + s), scale, s);
            const uint32_t hi = (s == p.L - 1) ? 0x10000u
                                               : mixture_cdf_u16<K>(cp.pi, cp.mu, cp.inv_s, __ldg(p.targets + s + 1),
                                                                    scale, s + 1);
            if (valid) p.intervals[P::BAND ? iv_elem<C>(p, n, c, q) : so] = lo | ((hi - 1u) << 16);
        }
        wg_sync(k);                                      // staging is rewritten by the next tile
    });
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
    const int planes = kind == 2 ? 2 : 1;
    const int kunits = kind == 0 ? p.Cin / 32 : p.Cin / 64;
    const long long M = (long long)p.N * p.H * p.W;
    const int w_plane = kunits * p.cout_pad * 128;
    const RingPlan r = plan_ring(kind == 1 ? conv_smem_cap() : SMEM_MAX, planes * w_plane + SMEM_RESERVE,
                                 planes * K1_A_BYTES, MAX_STAGES);
    L3C_REQUIRE(r.n_stages >= 1, "l3c_conv2d: weights of a %d -> %d 1x1 layer do not fit in shared memory", p.Cin, p.Cout);
    const CUtensorMapDataType dt = kind == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const int esz = kind == 0 ? 4 : 2, ch = kind == 0 ? 32 : 64;
    const void *x = kind == 0 ? (const void *)p.x : p.x_h, *w = kind == 0 ? (const void *)p.w : p.w_h;
    alignas(64) CUtensorMap map_x, map_w;
    if (!encode_tmap(&map_x, "l3c_conv2d", "x, 1x1", dt, x, {p.x_pitch, M}, {(long long)esz * p.x_pitch}, {ch, 64}) ||
        !encode_tmap(&map_w, "l3c_conv2d", "w, 1x1", dt, w, {ch, (long long)planes * kunits * p.cout_pad}, {128},
                     {ch, p.cout_pad}))
        return L3C_EINVAL;
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
    const char *name = kind == 0 ? "conv1x1_tf32_kernel" : kind == 1 ? "conv1x1_f16_kernel" : "conv1x1_f16x2_kernel";
#define L3C_1X1(K_, NB_)                                                                                          \
    if (kind == K_ && nb == NB_)                                                                                  \
    return launch_tc<conv1x1_tc_kernel<K_, NB_>>(name, grid_1x1(st, n_tiles), r.smem_bytes, st, map_x, map_w, q,  \
                                                 r.n_stages, n_tiles)
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
    const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const long long img[3] = {128, 128LL * p.W, 128LL * p.H * p.W};    // strides of the operand image
    alignas(64) CUtensorMap map_x, map_w;
    if (k3) {
        L3C_REQUIRE(p.Cout % 64 == 0, "l3c_conv2d[f16]: 3x3 layers need Cout %% 64 == 0 (got %d)", p.Cout);
        const bool ps = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
        L3C_REQUIRE(ps ? (p.y_pitch % 2 == 0 && p.y_coff % 2 == 0) : (p.y_pitch % 8 == 0 && p.y_coff % 8 == 0),
                    "l3c_conv2d[f16]: output pitch/offset alignment (pitch=%d coff=%d)", p.y_pitch, p.y_coff);
        L3C_REQUIRE(!(ps && p.residual), "l3c_conv2d[f16]: residual with pixel shuffle is not built");
        const int d = p.dilation;
        const int a_rows = TH + 2 * d, a_w = halo_w(d);
        L3C_REQUIRE(a_rows <= 256, "l3c_conv2d[f16]: dilation %d too large", d);
        const int a_bytes = a_rows * a_w * 128;          // one halo box = one stage = one tile
        // One stage per pipe: a second one (a tile of lookahead) measured no faster, and the 60 KB it takes at
        // d = 1 leave room on the SM for the CTAs of the other kernels that run beside this one in a codec step.
        const RingPlan r = plan_ring(conv_smem_cap(), W_RES_BYTES + SMEM_RESERVE, a_bytes, 1);
        L3C_REQUIRE(r.n_stages >= 1, "l3c_conv2d[f16]: halo of dilation %d does not fit in shared memory", d);
        if (!encode_tmap(&map_x, "l3c_conv2d[f16]", "x", dt, p.x_h, {64, p.W, p.H, p.N}, {img[0], img[1], img[2]},
                         {64, a_w, a_rows, 1}) ||
            !encode_tmap(&map_w, "l3c_conv2d[f16]", "w", dt, p.w_h, {64, 9LL * p.cout_pad}, {128}, {64, 64}))
            return L3C_EINVAL;
        const Params q = conv_params(p, p.H, p.W);
        const int ptiles = p.N * q.tiles_x * q.tiles_y;
        return launch_tc<conv_f16_kernel<0>>("conv3x3_f16_kernel", grid_3x3(st, p.cout_pad / 64, ptiles), r.smem_bytes,
                                             st, map_x, map_w, q, r.n_stages, a_bytes, ptiles);
    }
    // ---- 5x5 / stride 2
    L3C_REQUIRE(p.Cout % 64 == 0, "l3c_conv2d[f16]: 5x5/s2 layers need Cout %% 64 == 0 (got %d)", p.Cout);
    L3C_REQUIRE(!(p.flags & L3C_CONV_PIXEL_SHUFFLE2) && p.y_pitch % 8 == 0 && p.y_coff % 8 == 0,
                "l3c_conv2d[f16]: 5x5/s2 output pitch/offset alignment (pitch=%d coff=%d)", p.y_pitch, p.y_coff);
    const int Ho = (p.H + 4 - 5) / 2 + 1, Wo = (p.W + 4 - 5) / 2 + 1;
    // conv_smem_cap() >= 112 KB always leaves room for one stage per pipe; two from 178 KB
    const RingPlan r = plan_ring(conv_smem_cap(), SMEM_RESERVE, K5_STAGE_BYTES, 2);
    // element strides (2, 2): the box visits every second pixel / row; box sizes are given in traversed elements
    // (16 px -> 32, 10 rows -> 20)
    if (!encode_tmap(&map_x, "l3c_conv2d[f16]", "x, 5x5/s2", dt, p.x_h, {64, p.W, p.H, p.N}, {img[0], img[1], img[2]},
                     {64, 2 * TW, 20, 1}, {1, 2, 2, 1}) ||
        !encode_tmap(&map_w, "l3c_conv2d[f16]", "w, 5x5/s2", dt, p.w_h, {64, 25LL * p.cout_pad}, {128}, {64, 64}))
        return L3C_EINVAL;
    const Params q = conv_params(p, Ho, Wo);            // the epilogue works on OUTPUT pixels
    const int ptiles = p.N * q.tiles_x * q.tiles_y;
    return launch_tc<conv_f16_kernel<1>>("conv5x5s2_f16_kernel", grid_3x3(st, p.cout_pad / 64, ptiles), r.smem_bytes,
                                         st, map_x, map_w, q, r.n_stages, K5_STAGE_BYTES, ptiles);
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
    const int kchunks = Cin / 64;
    const long long M = (long long)N * HW;
    const int w_bytes = kchunks * npad * 128;
    const int stg_bytes = 2 * 64 * (npad + 1) * 4 + 64;
    const RingPlan r = plan_ring(conv_smem_cap(), w_bytes + stg_bytes + SMEM_RESERVE, K1_A_BYTES, MAX_STAGES);
    L3C_REQUIRE(r.n_stages >= 1, "l3c_lin_dmll_intervals: weights do not fit in shared memory (Cin=%d)", Cin);
    const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    alignas(64) CUtensorMap map_x, map_w;
    if (!encode_tmap(&map_x, "l3c_lin_dmll_intervals", "x", dt, x_h, {Cin, M}, {2LL * Cin}, {64, 64}) ||
        !encode_tmap(&map_w, "l3c_lin_dmll_intervals", "w", dt, w_h, {64, (long long)kchunks * npad}, {128}, {64, npad}))
        return L3C_EINVAL;
    ParamsLD q;
    q.bias = bias; q.sym = sym_dev; q.targets = targets_dev; q.intervals = intervals_dev;
    q.M = M; q.HW = HW; q.L = L; q.kchunks = kchunks; q.npad = npad;
    const int n_tiles = (int)((M + 63) / 64);
    const int grid = grid_1x1(st, n_tiles);
    if (rgb)
        return launch_tc<lin_dmll_f16_kernel<3, true, 2>>("lin_dmll_f16_kernel", grid, r.smem_bytes, st, map_x, map_w, q,
                                                          r.n_stages, n_tiles);
    return launch_tc<lin_dmll_f16_kernel<5, false, 3>>("lin_dmll_f16_kernel", grid, r.smem_bytes, st, map_x, map_w, q,
                                                       r.n_stages, n_tiles);
}

// l3c_lin_dmll_intervals for a band of a banded encode: rows [oy, oy + h) of the FP16 concat buffer x_h
// [N][Hl][W][Cin] of a full-width decoder window, the symbols of rows [y0, y0 + h) of the whole Hs x W plane sym_dev,
// the intervals in tile order to band stream planes [N][C][h * W]
extern "C" int l3c_lin_dmll_intervals_band(const void *x_h, int Hl, int oy, const void *w_h, const float *bias,
                                           const uint8_t *sym_dev, int Hs, int y0, int h, int W,
                                           const float *targets_dev, int N, int Cin, int C, int K, int L, int rgb,
                                           int th, int tw, uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    using namespace l3c::f16;
    L3C_REQUIRE(x_h && w_h && bias && sym_dev && targets_dev && intervals_dev,
                "l3c_lin_dmll_intervals_band: null pointer");
    L3C_REQUIRE(N >= 1 && N <= 65535 && Cin % 64 == 0 && Cin >= 64 && th >= 1 && tw >= 1,
                "l3c_lin_dmll_intervals_band: N=%d Cin=%d tile %dx%d", N, Cin, th, tw);
    L3C_REQUIRE(K == 10 && L >= 2 && L <= 256, "l3c_lin_dmll_intervals_band: K=%d L=%d (only K=10 is built)", K, L);
    L3C_REQUIRE((rgb && C == 3) || (!rgb && C == 5), "l3c_lin_dmll_intervals_band: built for RGB (C=3) and C=5 "
                                                     "bottlenecks, got C=%d rgb=%d", C, rgb);
    L3C_REQUIRE(h >= 1 && W >= 1 && (long long)h * W < (1ll << 31) && oy >= 0 && oy + h <= Hl && y0 >= 0 &&
                    y0 + h <= Hs,
                "l3c_lin_dmll_intervals_band: rows [%d, %d) of a %d-row window, [%d, %d) of a %d-row plane", oy,
                oy + h, Hl, y0, y0 + h, Hs);
    const int Kp = (rgb ? 4 : 3) * C * K;
    const int npad = (Kp + 63) / 64 * 64;
    cudaStream_t st = (cudaStream_t)stream;
    const int kchunks = Cin / 64;
    const int HW = h * W;
    const int tpi = (HW + 63) / 64;
    const long long n_tiles64 = (long long)N * tpi;
    L3C_REQUIRE(n_tiles64 < (1ll << 31), "l3c_lin_dmll_intervals_band: band too large");
    const int w_bytes = kchunks * npad * 128;
    const int stg_bytes = 2 * 64 * (npad + 1) * 4 + 64;
    const RingPlan r = plan_ring(conv_smem_cap(), w_bytes + stg_bytes + SMEM_RESERVE, K1_A_BYTES, MAX_STAGES);
    L3C_REQUIRE(r.n_stages >= 1, "l3c_lin_dmll_intervals_band: weights do not fit in shared memory (Cin=%d)", Cin);
    const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const __half *x0 = reinterpret_cast<const __half *>(x_h) + (long long)oy * W * Cin;
    alignas(64) CUtensorMap map_x, map_w;
    if (!encode_tmap(&map_x, "l3c_lin_dmll_intervals_band", "x", dt, x0, {Cin, HW, N},
                     {2LL * Cin, 2LL * Cin * Hl * W}, {64, 64, 1}) ||
        !encode_tmap(&map_w, "l3c_lin_dmll_intervals_band", "w", dt, w_h, {64, (long long)kchunks * npad}, {128},
                     {64, npad}))
        return L3C_EINVAL;
    ParamsLDBand q;
    q.bias = bias; q.sym = sym_dev; q.targets = targets_dev; q.intervals = intervals_dev;
    q.M = (long long)N * tpi * 64; q.HW = tpi * 64; q.L = L; q.kchunks = kchunks; q.npad = npad;
    q.g.sym_hw = (long long)Hs * W; q.g.l_hw = (long long)Hl * W;
    q.g.y0 = y0; q.g.h = h; q.g.W = W; q.g.Wl = W; q.g.oy = oy; q.g.ox = 0; q.g.th = th; q.g.tw = tw;
    q.tpi = tpi;
    const int n_tiles = (int)n_tiles64;
    const int grid = grid_1x1(st, n_tiles);
    if (rgb)
        return launch_tc<lin_dmll_f16_kernel<3, true, 2, ParamsLDBand>>("lin_dmll_band_f16_kernel", grid, r.smem_bytes,
                                                                        st, map_x, map_w, q, r.n_stages, n_tiles);
    return launch_tc<lin_dmll_f16_kernel<5, false, 3, ParamsLDBand>>("lin_dmll_band_f16_kernel", grid, r.smem_bytes,
                                                                     st, map_x, map_w, q, r.n_stages, n_tiles);
}
