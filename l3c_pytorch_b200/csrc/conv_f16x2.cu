// conv_f16x2.cu -- precision mode L3C_PREC_F16X2: the strict tensor-core mode.  Every operand x is carried as
// TWO FP16 numbers, hi = fp16(x) and lo = fp16((x - hi) * 2^11), so that x = hi + lo / 2^11 up to ~2^-22
// relative; a product is evaluated as
//        x * w  ~=  hi_x * hi_w  +  (hi_x * lo_w + lo_x * hi_w) / 2^11
// i.e. three wgmma (m64n64k16, FP16) per K step into TWO fp32 register accumulators (the dropped lo*lo term is
// 2^-22 relative); the epilogue combines acc1 + acc2 * 2^-11 in fp32.  This is the error-compensated split
// SURVEY.md section 7 asks for ("3xTF32"), built from FP16 pieces: fp32-class results (tests: rtol 2e-5 against
// PyTorch fp32, the tolerance of the CUDA-core kernel) at several times the FFMA rate, so that the one-scale RGB
// baselines and small images -- where the 10-bit operands of the fast mode cost more than 1e-4 bpsp -- also run
// on the tensor cores.
//
// Reference layers: the same as conv_f16.cu (3x3 / dilated 3x3 with 64 input channels, 1x1 with Cin % 64 == 0).
// Layouts: split operand image [N][H][W][2*C] FP16 (hi planes in channels [0,C), lo planes in [C,2C)); split
// weight image 3x3: [9 taps][cout_pad][128] (hi | lo), 1x1: [2*Cin/64 chunks: hi..., lo...][cout_pad][64].
// Kernel structure: conv_f16.cu's (weights resident, one halo box per filter column and plane, two consumer
// warpgroups on alternate tiles); one stage per pipe, one pipe for dilations > 1 (shared memory: 144 KB of weights
// + 40-64 KB per stage).  The 1x1 layers run conv1x1_tc_kernel<2, NB> (conv_f16.cu).
#include "tc_conv.cuh"

namespace l3c {
namespace f16x2 {
using namespace tcx;

constexpr int W_TAP_BYTES = 64 * 128;
constexpr int W_PLANE_BYTES = 9 * W_TAP_BYTES;        // 73728 per plane (hi / lo)

__global__ void __launch_bounds__(THREADS, 1)
conv3x3_f16x2_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                     const Params p, const int n_pipes, const int a_bytes, const int ptiles,
                     const TileSchedule ts) {
    L3C_TRACE_BEGIN;
    // [weights hi 72 KB][weights lo 72 KB][pipe 0: hi box, lo box][pipe 1: ...][barriers]
    const uint32_t w_base = smem_u32(smem_aligned());
    const uint32_t bars = w_base + 2 * W_PLANE_BYTES + n_pipes * 2 * a_bytes;
    pipeline_init(bars, &map_x, &map_w);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int k = warp < CONSUMER_WARPS ? warp >> 2 : warp - CONSUMER_WARPS;   // pipe
    if (k >= n_pipes) return;
    const int d = p.dilation;
    const int ct = blockIdx.y;
    const int lo_ch = 64;                                  // lo plane of a 64-channel operand image
    Ring ring(w_base + 2 * W_PLANE_BYTES, 2 * a_bytes, 1, bars, k);   // one stage (hi and lo box) per pipe
    TileQueue tiles(bars, k, n_pipes, ptiles, ts);

    if (warp >= CONSUMER_WARPS) {
        // ===================== TMA producer of pipe k =====================
        if (lane != 0) return;
        if (k == 0) {
            mbar_expect_tx(weight_bar(bars), 2 * W_PLANE_BYTES);
            for (int tap = 0; tap < 9; ++tap) {
                const int row = tap * (int)gridDim.y * 64 + ct * 64;
                tma_load_2d(w_base + tap * W_TAP_BYTES, &map_w, weight_bar(bars), 0, row);                      // hi
                tma_load_2d(w_base + W_PLANE_BYTES + tap * W_TAP_BYTES, &map_w, weight_bar(bars), 64, row);     // lo
            }
        }
        produce_tiles(tiles, [&](int t) {
            const Tile c = tile_of(p, t);
            for (int dx = 0; dx < 3; ++dx) {
                const Slot s = ring.acquire(2 * a_bytes);
                tma_load_4d(s.dst, &map_x, s.bar, 0, c.tx * TW + (dx - 1) * d, c.ty * TH - d, c.n);
                tma_load_4d(s.dst + a_bytes, &map_x, s.bar, lo_ch, c.tx * TW + (dx - 1) * d, c.ty * TH - d, c.n);
            }
        });
        return;
    }

    // ===================== consumer warpgroup k: wgmma + epilogue =====================
    const int w = warp & 3;
    mbar_wait(weight_bar(bars), 0);
    consume_tiles(tiles, [&](int t) {
        const Tile c = tile_of(p, t);
        float acc1[2][32], acc2[2][32];                   // hi*hi | hi*lo + lo*hi; rows 0..63 / 64..127
#pragma unroll
        for (int h = 0; h < 2; ++h) { acc_zero(acc1[h]); acc_zero(acc2[h]); }
        for (int dx = 0; dx < 3; ++dx) {
            const uint32_t a_base = ring.wait();
            wgmma_fence();
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {
                const uint64_t bh = make_desc(w_base + (dy * 3 + dx) * W_TAP_BYTES);
                const uint64_t bl = make_desc(w_base + W_PLANE_BYTES + (dy * 3 + dx) * W_TAP_BYTES);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t ah = make_desc(a_base + (dy * d * TW + 64 * h) * 128);
                    const uint64_t al = make_desc(a_base + a_bytes + (dy * d * TW + 64 * h) * 128);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const uint32_t first = (dx | dy | kk) != 0 ? 1u : 0u;
                        wgmma_f16(acc1[h], ah + 2u * kk, bh + 2u * kk, first);        // hi * hi
                        wgmma_f16(acc2[h], ah + 2u * kk, bl + 2u * kk, first);        // hi * lo
                        wgmma_f16(acc2[h], al + 2u * kk, bh + 2u * kk, 1u);           // lo * hi
                    }
                }
            }
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int h = 0; h < 2; ++h) { acc_fence(acc1[h]); acc_fence(acc2[h]); }
            ring.release();
        }
        // x = hi*hi + (hi*lo + lo*hi) / 2^11: combined before the epilogue, so that acc2 is dead there
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) acc1[h][i] = __fmaf_rn(acc2[h][i], LO_INV, acc1[h][i]);
        image_epilogue<true, Halves::ROWS>(p, c, ct, w, acc1);
    });
}

// fp32 [n_px][C] -> split image [n_px][2*C]: for the activations that CUDA-core layers (5x5/s2, Cin = 3 / 5)
// produce in this mode and for callers that feed a tensor-core layer from outside the network
__global__ void split_kernel(const float4 *__restrict__ x, __half *__restrict__ out, long long n4, int C) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = __ldg(x + i);
    const long long e = i * 4, px = e / C;
    const int c = (int)(e - px * C);
    uint32_t h0, l0, h1, l1;
    split_h2(v.x, v.y, h0, l0);
    split_h2(v.z, v.w, h1, l1);
    __half *o = out + px * 2 * C + c;
    *reinterpret_cast<uint2 *>(o) = make_uint2(h0, h1);
    *reinterpret_cast<uint2 *>(o + C) = make_uint2(l0, l1);
}

}  // namespace f16x2

extern "C" int l3c_split_f16x2(const float *x, long long n_px, int C, void *out, void *stream) {
    L3C_REQUIRE(x && out && n_px >= 0 && C >= 4 && C % 4 == 0, "l3c_split_f16x2: bad arguments (n_px=%lld C=%d)", n_px, C);
    const long long n4 = n_px * C / 4;
    if (n4 == 0) return L3C_OK;
    f16x2::split_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4 *>(x), reinterpret_cast<__half *>(out), n4, C);
    L3C_LAUNCH_CHECK("split_f16x2_kernel");
    return L3C_OK;
}

// x_h: split operand image [N][H][W][x_pitch = 2*Cin] (hi | lo); w_h: split weight image (engine.PackedConv.get_f16x2)
int conv2d_f16x2(const l3c_conv_t &p, cudaStream_t st) {
    using namespace f16x2;
    const bool k3 = p.ksize == 3 && p.stride == 1 && p.Cin == 64 && p.x_pitch == 128;
    const bool k1 = p.ksize == 1 && p.stride == 1 && p.Cin % 64 == 0 && p.x_pitch == 2 * p.Cin &&
                    !(p.flags & L3C_CONV_PIXEL_SHUFFLE2);
    L3C_REQUIRE(k3 || k1, "l3c_conv2d[f16x2]: tensor-core path needs 3x3/s1/Cin=64 or 1x1/Cin%%64==0 on split operand "
                          "images (got k=%d s=%d Cin=%d pitch=%d)", p.ksize, p.stride, p.Cin, p.x_pitch);
    L3C_REQUIRE(p.x_h && p.w_h && (p.y || p.y_h), "l3c_conv2d[f16x2]: x_h / w_h and an output are required");
    L3C_REQUIRE(p.cout_pad % 64 == 0 && p.cout_pad >= p.Cout, "l3c_conv2d[f16x2]: cout_pad=%d", p.cout_pad);
    L3C_REQUIRE(!(p.flags & ~(L3C_CONV_RELU | L3C_CONV_PIXEL_SHUFFLE2)), "l3c_conv2d[f16x2]: unsupported flags %u", p.flags);
    if (k3) {
        L3C_REQUIRE(p.Cout % 64 == 0, "l3c_conv2d[f16x2]: 3x3 layers need Cout %% 64 == 0 (got %d)", p.Cout);
        const bool ps = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
        L3C_REQUIRE(!(ps && p.residual), "l3c_conv2d[f16x2]: residual with pixel shuffle is not built");
        L3C_REQUIRE(!p.y_h || (p.yh_pitch > 0 && p.yh_lo_off > 0 && p.yh_pitch % 8 == 0 && p.yh_lo_off % 8 == 0),
                    "l3c_conv2d[f16x2]: the split output image needs yh_pitch / yh_lo_off (multiples of 8)");
        L3C_REQUIRE(ps ? (p.y_pitch % 2 == 0 && p.y_coff % 2 == 0) : (p.y_pitch % 8 == 0 && p.y_coff % 8 == 0),
                    "l3c_conv2d[f16x2]: output pitch/offset alignment (pitch=%d coff=%d)", p.y_pitch, p.y_coff);
        const int d = p.dilation;
        const int a_rows = TH + 2 * d;
        const int a_bytes = a_rows * TW * 128;
        const RingPlan r = plan_ring(SMEM_MAX, 2 * W_PLANE_BYTES + SMEM_RESERVE, 2 * a_bytes, 1, true);
        L3C_REQUIRE(r.n_stages >= 1, "l3c_conv2d[f16x2]: halo of dilation %d does not fit in shared memory", d);
        alignas(64) CUtensorMap map_x, map_w;
        if (!encode_tmap(&map_x, "l3c_conv2d[f16x2]", "x", CU_TENSOR_MAP_DATA_TYPE_FLOAT16, p.x_h, {128, p.W, p.H, p.N},
                         {256, 256LL * p.W, 256LL * p.H * p.W}, {64, TW, a_rows, 1}) ||
            !encode_tmap(&map_w, "l3c_conv2d[f16x2]", "w", CU_TENSOR_MAP_DATA_TYPE_FLOAT16, p.w_h, {128, 9LL * p.cout_pad},
                         {256}, {64, 64}))
            return L3C_EINVAL;
        const Params q = conv_params(p, p.H, p.W);
        const int ptiles = p.N * q.tiles_x * q.tiles_y;
        return launch_tc<conv3x3_f16x2_kernel>("conv3x3_f16x2_kernel", grid_3x3(st, p.cout_pad / 64, ptiles),
                                               r.smem_bytes, st, map_x, map_w, q, r.n_pipes, a_bytes, ptiles);
    }
    return conv1x1_tc(p, st);
}

}  // namespace l3c
