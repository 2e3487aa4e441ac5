// conv_tf32.cu -- precision mode L3C_PREC_TF32: the 3x3 (optionally dilated) 64-input-channel convolutions as
// implicit GEMMs on the Hopper tensor cores: TMA (cp.async.bulk.tensor) stages shifted NHWC windows into
// 128B-swizzled shared memory, a consumer warpgroup issues wgmma (m64n64k8, tf32) for the two 64-pixel halves of
// an 8x16-pixel tile, keeps the fp32 accumulators in registers and fuses bias / ReLU / residual / channel slice /
// PixelShuffle(2) into its epilogue.  The 1x1 layers of this mode run conv1x1_tc_kernel (conv_f16.cu).
//
// Reference layers this replaces: every `default_conv(64, Cout, 3, rate=r)` of the L3C stack
// (pytorch_ext.py:57-61; ResBlock edsr.py:63-89, body-final conv net.py:110,170, Head head.py:49-56,
// Upsampler edsr.py:92-101, atrous convs prob_clf.py:54-55) -- cuDNN fp32 in the reference.
//
// Implicit GEMM mapping (per 8x16-pixel tile, per filter tap t=(ky,kx)):
//   A[m][k] = x[n, ty0 + m/16 + (ky-1)*d, tx0 + m%16 + (kx-1)*d, k]   (zero outside the image: TMA
//             out-of-bounds fill implements the conv padding), m = 0..127, k = 0..63
//   B[n][k] = w[n, k, ky, kx]                                          n = 0..63 (one Cout tile)
// The 9 x 2 weight slabs of the CTA's Cout tile (144 KB) stay in shared memory; for each filter column dx and
// K-half ONE box of (8 + 2d) rows x 16 pixels x 32 channels is staged, and the three dy taps read it at row
// offsets dy*d*16 pixels (multiples of the 1024 B swizzle atom).
// Accumulation order per output element: (dx, K-half, dy, k-step) -- fixed, independent of batch, image size,
// tile position and pipe: encoder-side and decoder-side evaluations are bit-identical.
//
// Precision: the tensor core reads only the upper 19 bits of each fp32 operand (truncation), which measurably
// biases the bit cost.  Operands are therefore pre-rounded to TF32 with round-to-nearest: weights once on the
// host side, activations by the producing layer's epilogue, which writes a second, rounded copy (`y_tf32`) next
// to the fp32 tensor that residual adds and the fp32 layers keep using.
// (The faster FP16-operand variant of this path is conv_f16.cu, precision L3C_PREC_F16.)
#include <mutex>

#include "tc_conv.cuh"

namespace l3c {

namespace tc {
using namespace tcx;

constexpr int B_HALF = 64 * 128;               // 64 cout rows x 128 B (32 fp32 channels)
constexpr int W_RES_BYTES = 9 * 2 * B_HALF;    // 147456

__global__ void __launch_bounds__(THREADS, 1)
conv3x3_tf32_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const Params p, const int n_pipes, const int n_stages, const int a_bytes, const int ptiles,
                    const TileSchedule ts) {
    L3C_TRACE_BEGIN;
    // [weights 144 KB][pipe 0 stages][pipe 1 stages][barriers]
    const uint32_t w_base = smem_u32(smem_aligned());
    const uint32_t bars = w_base + W_RES_BYTES + n_pipes * n_stages * a_bytes;
    pipeline_init(bars, &map_x, &map_w);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k = warp < CONSUMER_WARPS ? warp >> 2 : warp - CONSUMER_WARPS;   // pipe
    if (k >= n_pipes) return;
    const int d = p.dilation;
    const int ct = blockIdx.y;                        // this CTA's Cout tile (weights stay resident)
    Ring ring(w_base + W_RES_BYTES, a_bytes, n_stages, bars, k);
    TileQueue tiles(bars, k, n_pipes, ptiles, ts);

    if (warp >= CONSUMER_WARPS) {
        // ===================== TMA producer of pipe k =====================
        if (lane != 0) return;
        if (k == 0) {
            mbar_expect_tx(weight_bar(bars), W_RES_BYTES);
            for (int slab = 0; slab < 18; ++slab)     // slab = tap*2 + K-half; rows [slab][cout_pad]
                tma_load_2d(w_base + slab * B_HALF, &map_w, weight_bar(bars), 0, slab * (int)gridDim.y * 64 + ct * 64);
        }
        produce_tiles(tiles, [&](int t) {
            const Tile c = tile_of(p, t);
            for (int unit = 0; unit < 6; ++unit) {    // unit = dx*2 + K-half
                const Slot s = ring.acquire(a_bytes);
                tma_load_4d(s.dst, &map_x, s.bar, (unit & 1) * 32, c.tx * TW + ((unit >> 1) - 1) * d, c.ty * TH - d, c.n);
            }
        });
        return;
    }

    // ===================== consumer warpgroup k: wgmma + epilogue =====================
    const int w = warp & 3;
    const int tq = lane & 3, tr = lane >> 2;              // column pair / row inside the fragment
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool shuffle = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
    const bool round_y = (p.flags & L3C_CONV_ROUND_TF32) != 0;
    mbar_wait(weight_bar(bars), 0);
    consume_tiles(tiles, [&](int t) {
        const Tile c = tile_of(p, t);
        float acc[2][32];                                 // rows 0..63 / 64..127 of the tile
        acc_zero(acc[0]);
        acc_zero(acc[1]);
        for (int unit = 0; unit < 6; ++unit) {
            const int dx = unit >> 1, kh = unit & 1;
            const uint32_t a0 = ring.wait();
            wgmma_fence();
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {
                const uint64_t db = make_desc(w_base + ((dy * 3 + dx) * 2 + kh) * B_HALF);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t da = make_desc(a0 + (dy * d * TW + 64 * h) * 128);   // dy*d rows of 16 px
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)       // +32 B (8 tf32) along K inside the 128 B swizzle row
                        wgmma_tf32(acc[h], da + 2u * kk, db + 2u * kk, (unit | dy | kk) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            wgmma_wait0();
            acc_fence(acc[0]);
            acc_fence(acc[1]);
            ring.release();
        }
        // epilogue: element pairs, so that y and its TF32 twin need no transpose; fragment (h, column half cc) =
        // tile row 4h + w, pixels tr / tr + 8, columns 32cc + 8jb + 2tq
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int oy = c.ty * TH + 4 * h + w;
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
                const float *v = acc[h] + 16 * cc;
#pragma unroll
                for (int rh = 0; rh < 2; ++rh) {
                    const int ox = c.tx * TW + tr + 8 * rh;
                    if (oy >= p.H || ox >= p.W) continue;
                    const size_t pix = ((size_t)c.n * p.H + oy) * p.W + ox;
#pragma unroll
                    for (int jb = 0; jb < 4; ++jb) {
                        const int co = ct * 64 + 32 * cc + 8 * jb + 2 * tq;
                        const float2 bb = __ldg(reinterpret_cast<const float2 *>(p.bias + co));
                        float a = v[4 * jb + 2 * rh] + bb.x;
                        float b = v[4 * jb + 2 * rh + 1] + bb.y;
                        if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                        if (!shuffle) {
                            const size_t off = pix * p.y_pitch + p.y_coff + co;
                            if (p.residual) {
                                const float2 r = __ldg(reinterpret_cast<const float2 *>(p.residual + off));
                                a += r.x; b += r.y;
                            }
                            if (p.y_tf32) *reinterpret_cast<float2 *>(p.y_tf32 + off) = make_float2(round_tf32(a), round_tf32(b));
                            if (round_y) { a = round_tf32(a); b = round_tf32(b); }
                            *reinterpret_cast<float2 *>(p.y + off) = make_float2(a, b);
                        } else {
                            // out[n, 2*oy+i, 2*ox+jj, cq] = conv[n, oy, ox, 4*cq + 2*i + jj]; co is even:
                            // (co, co+1) -> same cq and i, jj = 0 / 1 -> two horizontally adjacent pixels
                            const int cq = co >> 2, si = (co >> 1) & 1;
                            const size_t o2 = (((size_t)c.n * (2 * p.H) + 2 * oy + si) * (2 * p.W) + 2 * ox) * p.y_pitch +
                                              p.y_coff + cq;
                            if (p.y_tf32) { p.y_tf32[o2] = round_tf32(a); p.y_tf32[o2 + p.y_pitch] = round_tf32(b); }
                            if (round_y) { a = round_tf32(a); b = round_tf32(b); }
                            p.y[o2] = a;
                            p.y[o2 + p.y_pitch] = b;
                        }
                    }
                }
            }
        }
    });
}

// A checked 3x3 layer: p.x is read as N x H x W pixels of p.Cin = 64 channels, p.x_pitch apart
static int launch_3x3(const l3c_conv_t &p, cudaStream_t st) {
    const int d = p.dilation;
    const int a_rows = TH + 2 * d;
    const int a_bytes = a_rows * TW * 128;
    const RingPlan r = plan_ring(SMEM_MAX, W_RES_BYTES + SMEM_RESERVE, a_bytes, 2, true);
    L3C_REQUIRE(a_rows <= 256 && r.n_stages >= 1, "l3c_conv2d[tf32]: halo of dilation %d does not fit in shared memory", d);

    // tensor-core weight image: [tap][K-half = Cin/32][cout_pad][32] fp32 (engine.PackedConv.get_tc)
    alignas(64) CUtensorMap map_x, map_w;
    if (!encode_tmap(&map_x, "l3c_conv2d[tf32]", "x", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.x, {p.Cin, p.W, p.H, p.N},
                     {4LL * p.x_pitch, 4LL * p.W * p.x_pitch, 4LL * p.H * p.W * p.x_pitch}, {32, TW, a_rows, 1}) ||
        !encode_tmap(&map_w, "l3c_conv2d[tf32]", "w", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.w, {32, 18LL * p.cout_pad},
                     {128}, {32, 64}))
        return L3C_EINVAL;
    const Params q = conv_params(p, p.H, p.W);
    const int ptiles = p.N * q.tiles_x * q.tiles_y;
    return launch_tc<conv3x3_tf32_kernel>("conv3x3_tf32_kernel", grid_3x3(st, p.cout_pad / 64, ptiles), r.smem_bytes,
                                          st, map_x, map_w, q, r.n_pipes, r.n_stages, a_bytes, ptiles);
}

}  // namespace tc

int conv2d_tf32(const l3c_conv_t &p, cudaStream_t st) {
    using namespace tc;
    if (p.precision != L3C_PREC_TF32) {
        set_error("l3c_conv2d: precision mode %d is not built (available: fp32, tf32, f16, f16x2)", p.precision);
        return L3C_EINVAL;
    }
    // The tensor-core kernels cover the 3x3 / 64-input-channel layers (> 92 % of the FLOPs of a round trip) and
    // the 1x1 layers with Cin % 64 == 0.  The host mirror routes the other layers (5x5/s2 down-sampling,
    // Cin != 64) to L3C_PREC_FP32 explicitly (engine.conv2d); nothing falls back silently here.
    const bool k3 = p.ksize == 3 && p.stride == 1 && p.Cin == 64 && p.x_pitch == 64;
    const bool k1 = p.ksize == 1 && p.stride == 1 && p.Cin % 64 == 0 && p.x_pitch == p.Cin &&
                    !(p.flags & L3C_CONV_PIXEL_SHUFFLE2);
    const bool eligible = (k3 || k1) && p.cout_pad % 64 == 0 && p.cout_pad >= p.Cout &&
                          (k1 || ((p.Cout % 64 == 0) && (p.y_pitch % 4 == 0) && (p.y_coff % 4 == 0)));
    L3C_REQUIRE(eligible, "l3c_conv2d: tf32 tensor-core path needs 3x3/Cin=64 or 1x1/Cin%%64==0, stride 1 "
                          "(got k=%d s=%d Cin=%d pitch=%d Cout=%d)", p.ksize, p.stride, p.Cin, p.x_pitch, p.Cout);
    if (k1) return conv1x1_tc(p, st);
    return tc::launch_3x3(p, st);
}

// The zero bias of the data-gradient launches: 64 floats per device, made once
static int zero_bias(const float **out) {
    static std::mutex mu;
    static float *buf[64] = {};
    std::lock_guard<std::mutex> lk(mu);
    float *&b = buf[current_device_slot()];
    if (!b) {
        L3C_CUDA(cudaMalloc(&b, 64 * sizeof(float)));
        L3C_CUDA(cudaMemset(b, 0, 64 * sizeof(float)));
        L3C_CUDA(cudaDeviceSynchronize());
    }
    *out = b;
    return L3C_OK;
}

}  // namespace l3c

using namespace l3c;

extern "C" int l3c_conv3x3_dgrad(const float *dy_dev, const float *w_dev, int N, int H, int W, int Cin, int Cout,
                                 int dilation, float *dx_dev, void *stream) {
    if (int e = conv3x3_backward_args("l3c_conv3x3_dgrad", {dy_dev, w_dev, dx_dev}, N, H, W, Cin, Cout, dilation))
        return e;
    const float *zero = nullptr;
    if (int e = zero_bias(&zero)) return e;
    // slice s: the 64 channels 64s.. of dy (pitch Cout) against image slice s, added to dx through the residual
    for (int s = 0; s < Cout / 64; ++s) {
        l3c_conv_t p = {};
        p.x = dy_dev + 64 * s;
        p.w = w_dev + (size_t)s * 9 * 2 * 64 * 32;
        p.bias = zero;
        p.residual = s ? dx_dev : nullptr;
        p.y = dx_dev;
        p.N = N; p.H = H; p.W = W;
        p.Cin = 64; p.x_pitch = Cout;
        p.Cout = 64; p.cout_pad = 64; p.y_pitch = 64; p.y_coff = 0;
        p.ksize = 3; p.stride = 1; p.dilation = dilation;
        p.flags = 0; p.precision = L3C_PREC_TF32;
        if (int e = tc::launch_3x3(p, (cudaStream_t)stream)) return e;
    }
    return L3C_OK;
}
