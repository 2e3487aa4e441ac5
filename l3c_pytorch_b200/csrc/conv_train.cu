// conv_train.cu -- backward of the 3x3 / stride-1 / 64-input-channel convolutions of the training step (DESIGN §4.11):
// the weight and bias gradient (conv3x3_wgrad_kernel + conv3x3_wgrad_finish_kernel), the TF32 rounding of operand
// images (round_tf32_kernel) and the argument checks both backward passes share.  The data gradient runs the forward
// kernel conv3x3_tf32_kernel on a flipped weight image (l3c_conv3x3_dgrad, conv_tf32.cu).
//
// Weight gradient as a GEMM: M = Cout (one 64-row tile per blockIdx.y), N = 9 taps x 64 ci, K = the pixels.
//   dW[co][tap][ci] = sum_p dy[p][co] * x[p + d (ky - 1, kx - 1)][ci]
// Both operands are stored pixel-major (NHWC), so K is their outer index; TF32 wgmma takes only K-major operands from
// shared memory, so this kernel uses mma.sync m16n8k8 with fragments loaded from row-padded shared memory instead.
// Per 8x16-pixel tile the CTA stages dy [128 px][64 co] and the x halo [(8 + 2d) x (16 + 2d) px][64 ci], both rounded
// to TF32 (cvt.rna) on the way in and zero outside the image; warp w (9 of them) owns tap w and keeps its
// [64 co][64 ci] accumulators in registers across all tiles of the CTA's chunk.
// Accumulation order of a dW element: chunk by chunk in chunk order (finish kernel); inside a chunk tile by tile,
// inside a tile k-step by k-step (8 pixels each, in raster order) -- fixed by the shape alone.
#include "common.cuh"
#include "tc_ptx.cuh"

namespace l3c {

constexpr int64_t MAX_PLANE_PIXELS = 1ll << 30;     // codec.MAX_PLANE_PIXELS

int conv3x3_backward_args(const char *fn, std::initializer_list<const void *> ptrs, int N, int H, int W, int Cin,
                          int Cout, int dilation) {
    for (const void *p : ptrs) {
        L3C_REQUIRE(p != nullptr, "%s: null pointer", fn);
        L3C_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15u) == 0, "%s: pointer %p is not 16-byte aligned", fn, p);
    }
    L3C_REQUIRE(Cin == 64, "%s: Cin=%d (the backward kernels take 64 input channels)", fn, Cin);
    L3C_REQUIRE(Cout == 64 || Cout == 256, "%s: Cout=%d (64 or 256)", fn, Cout);
    L3C_REQUIRE(dilation == 1 || dilation == 2 || dilation == 4, "%s: dilation=%d (1, 2 or 4)", fn, dilation);
    L3C_REQUIRE(N >= 1 && N <= 65535 && H >= 1 && W >= 1, "%s: N=%d H=%d W=%d", fn, N, H, W);
    L3C_REQUIRE((int64_t)H * W <= MAX_PLANE_PIXELS, "%s: a %dx%d plane is above %lld pixels", fn, H, W,
                (long long)MAX_PLANE_PIXELS);
    return L3C_OK;
}

namespace wg {
using tcx::round_tf32;

constexpr int TH = 8, TW = 16, TP = TH * TW;   // pixel tile
constexpr int PITCH = 72;       // floats per staged pixel: lanes (g, q) of a fragment load hit banks 8q + g
constexpr int WARPS = 9, THREADS = 32 * WARPS;
constexpr int LOADERS = THREADS / 16;          // pixels staged per pass (16 threads of float4 per pixel)
constexpr int TARGET_CTAS = 132;               // chunks x Cout tiles; a constant, so the split follows the shape only
constexpr int NCOL = 9 * 64;                   // dW columns of one output channel: tap * 64 + ci

struct Params {
    const float *x, *dy;
    float *part;            // [n_chunks][Cout][NCOL] partial dW, then [n_chunks][Cout] partial db
    int H, W, Cout, d, tiles_x, tiles_y, n_chunks;
    int64_t n_tiles, tiles_per_chunk;
};

struct Plan {
    int tiles_x, tiles_y, n_chunks;
    int64_t n_tiles, tiles_per_chunk;
};

static Plan plan(int N, int H, int W, int Cout) {
    Plan r;
    r.tiles_x = ceil_div(W, TW);
    r.tiles_y = ceil_div(H, TH);
    r.n_tiles = (int64_t)N * r.tiles_x * r.tiles_y;
    const int per_ct = TARGET_CTAS / (Cout / 64) > 1 ? TARGET_CTAS / (Cout / 64) : 1;
    r.tiles_per_chunk = ceil_div64(r.n_tiles, per_ct);
    r.n_chunks = (int)ceil_div64(r.n_tiles, r.tiles_per_chunk);
    return r;
}

static int64_t work_bytes(const Plan &r, int Cout) { return (int64_t)r.n_chunks * Cout * (NCOL + 1) * 4; }

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ float4 round4(float4 v) {
    return make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
}

__global__ void __launch_bounds__(THREADS, 1) conv3x3_wgrad_kernel(const Params p) {
    extern __shared__ float4 smem4[];
    float *dys = reinterpret_cast<float *>(smem4);        // [TP][PITCH]
    float *xs = dys + TP * PITCH;                          // [(TH + 2d) (TW + 2d)][PITCH]
    const int d = p.d, hw = TW + 2 * d, hh = TH + 2 * d;
    const int ct = blockIdx.y, chunk = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ky = warp / 3, kx = warp % 3;                // this warp's tap
    const int g = lane >> 2, q = lane & 3;                 // fragment row group / thread in group
    const int qd = tid & 15;                               // the channel quad this thread stages
    float acc[4][8][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
    float4 dbacc = make_float4(0.f, 0.f, 0.f, 0.f);       // dy sum of channels 4qd.. over this thread's pixels

    const int64_t t0 = (int64_t)chunk * p.tiles_per_chunk;
    const int64_t t1 = t0 + p.tiles_per_chunk < p.n_tiles ? t0 + p.tiles_per_chunk : p.n_tiles;
    for (int64_t t = t0; t < t1; ++t) {
        const int tx = (int)(t % p.tiles_x);
        const int64_t rest = t / p.tiles_x;
        const int ty = (int)(rest % p.tiles_y);
        const int64_t n = rest / p.tiles_y;
        __syncthreads();                                   // the previous tile's fragments are read
        for (int px = tid >> 4; px < TP; px += LOADERS) {
            const int oy = ty * TH + px / TW, ox = tx * TW + px % TW;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (oy < p.H && ox < p.W)
                v = __ldg(reinterpret_cast<const float4 *>(p.dy + ((n * p.H + oy) * p.W + ox) * p.Cout + ct * 64 + 4 * qd));
            dbacc.x += v.x; dbacc.y += v.y; dbacc.z += v.z; dbacc.w += v.w;
            *reinterpret_cast<float4 *>(dys + px * PITCH + 4 * qd) = round4(v);
        }
        for (int hp = tid >> 4; hp < hh * hw; hp += LOADERS) {
            const int iy = ty * TH - d + hp / hw, ix = tx * TW - d + hp % hw;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
                v = __ldg(reinterpret_cast<const float4 *>(p.x + ((n * p.H + iy) * p.W + ix) * 64 + 4 * qd));
            *reinterpret_cast<float4 *>(xs + hp * PITCH + 4 * qd) = round4(v);
        }
        __syncthreads();
#pragma unroll 2
        for (int ks = 0; ks < TP / 8; ++ks) {              // 8 pixels of one tile row per k-step
            const int row = ks >> 1, c0 = (ks & 1) * 8;
            // A[m = co][k = px] = dy[px][co]; B[k = px][n = ci] = x[px shifted by the tap][ci]
            const float *pa = dys + (ks * 8 + q) * PITCH + g;
            const float *pb = xs + ((row + ky * d) * hw + c0 + kx * d + q) * PITCH + g;
            uint32_t a[4][4], b[8][2];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) {
                a[mt][0] = __float_as_uint(pa[16 * mt]);
                a[mt][1] = __float_as_uint(pa[16 * mt + 8]);
                a[mt][2] = __float_as_uint(pa[4 * PITCH + 16 * mt]);
                a[mt][3] = __float_as_uint(pa[4 * PITCH + 16 * mt + 8]);
            }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                b[nt][0] = __float_as_uint(pb[8 * nt]);
                b[nt][1] = __float_as_uint(pb[4 * PITCH + 8 * nt]);
            }
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) mma_tf32(acc[mt][nt], a[mt], b[nt]);
        }
    }
    // partial dW of this chunk; fragment (mt, nt): rows co = 16 mt + g (+ 8), columns ci = 8 nt + 2 q (+ 1)
    float *pw = p.part + (size_t)chunk * p.Cout * NCOL;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const size_t off = (size_t)(ct * 64 + 16 * mt + g) * NCOL + warp * 64 + 8 * nt + 2 * q;
            *reinterpret_cast<float2 *>(pw + off) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
            *reinterpret_cast<float2 *>(pw + off + 8 * NCOL) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
        }
    // partial db: the LOADERS threads of each channel quad, in thread order
    __syncthreads();
    float4 *red = smem4;
    red[tid] = dbacc;
    __syncthreads();
    if (tid < 64) {
        float s = 0.f;
        for (int j = 0; j < LOADERS; ++j) {
            const float4 v = red[j * 16 + (tid >> 2)];
            s += (tid & 3) == 0 ? v.x : (tid & 3) == 1 ? v.y : (tid & 3) == 2 ? v.z : v.w;
        }
        p.part[(size_t)p.n_chunks * p.Cout * NCOL + (size_t)chunk * p.Cout + ct * 64 + tid] = s;
    }
}

// dW and db: the chunks' partial sums in chunk order; dW written OIHW ([co][ci][ky][kx])
__global__ void conv3x3_wgrad_finish_kernel(const float *__restrict__ part, int n_chunks, int Cout,
                                            float *__restrict__ dw, float *__restrict__ db) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nw = Cout * NCOL;
    if (i < nw) {
        float s = 0.f;
        for (int c = 0; c < n_chunks; ++c) s += part[(size_t)c * nw + i];
        const int co = i / NCOL, tap = (i % NCOL) / 64, ci = i % 64;
        dw[(co * 64 + ci) * 9 + tap] = s;
    } else if (i < nw + Cout) {
        const int co = i - nw;
        float s = 0.f;
        for (int c = 0; c < n_chunks; ++c) s += part[(size_t)n_chunks * nw + (size_t)c * Cout + co];
        db[co] = s;
    }
}

__global__ void round_tf32_kernel(const float *__restrict__ x, float *y, int64_t n) {
    const int64_t n4 = n / 4, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
        reinterpret_cast<float4 *>(y)[i] = round4(__ldg(reinterpret_cast<const float4 *>(x) + i));
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) y[4 * n4 + threadIdx.x] = round_tf32(x[4 * n4 + threadIdx.x]);
}

}  // namespace wg
}  // namespace l3c

using namespace l3c;

extern "C" int l3c_round_tf32(const float *x_dev, float *y_dev, int64_t n, void *stream) {
    L3C_REQUIRE(x_dev && y_dev, "l3c_round_tf32: null pointer");
    L3C_REQUIRE(((reinterpret_cast<uintptr_t>(x_dev) | reinterpret_cast<uintptr_t>(y_dev)) & 15u) == 0,
                "l3c_round_tf32: pointers must be 16-byte aligned");
    L3C_REQUIRE(n >= 0, "l3c_round_tf32: n=%lld", (long long)n);
    if (n == 0) return L3C_OK;
    const int64_t blocks = ceil_div64(n / 4 + 1, 256);
    wg::round_tf32_kernel<<<(unsigned)(blocks < 4 * sm_count() ? blocks : 4 * sm_count()), 256, 0,
                            (cudaStream_t)stream>>>(x_dev, y_dev, n);
    L3C_LAUNCH_CHECK("round_tf32_kernel");
    return L3C_OK;
}

extern "C" int64_t l3c_conv3x3_wgrad_workspace(int N, int H, int W, int Cout) {
    if (N < 1 || N > 65535 || H < 1 || W < 1 || (int64_t)H * W > MAX_PLANE_PIXELS || (Cout != 64 && Cout != 256))
        return 0;
    return wg::work_bytes(wg::plan(N, H, W, Cout), Cout);
}

extern "C" int l3c_conv3x3_wgrad(const float *x_dev, const float *dy_dev, int N, int H, int W, int Cin, int Cout,
                                 int dilation, float *dw_dev, float *db_dev, float *work_dev, int64_t work_bytes,
                                 void *stream) {
    using namespace wg;
    if (int e = conv3x3_backward_args("l3c_conv3x3_wgrad", {x_dev, dy_dev, dw_dev, db_dev, work_dev}, N, H, W, Cin,
                                      Cout, dilation))
        return e;
    const Plan r = plan(N, H, W, Cout);
    L3C_REQUIRE(work_bytes >= wg::work_bytes(r, Cout), "l3c_conv3x3_wgrad: workspace of %lld bytes, %lld needed",
                (long long)work_bytes, (long long)wg::work_bytes(r, Cout));
    cudaStream_t st = (cudaStream_t)stream;
    const int smem = (TP + (TH + 2 * dilation) * (TW + 2 * dilation)) * PITCH * 4;
    static bool configured_dev[64] = {};
    bool &configured = configured_dev[current_device_slot()];
    if (!configured) {
        L3C_CUDA(cudaFuncSetAttribute(conv3x3_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (TP + (TH + 8) * (TW + 8)) * PITCH * 4));
        configured = true;
    }
    Params p;
    p.x = x_dev; p.dy = dy_dev; p.part = work_dev;
    p.H = H; p.W = W; p.Cout = Cout; p.d = dilation;
    p.tiles_x = r.tiles_x; p.tiles_y = r.tiles_y; p.n_chunks = r.n_chunks;
    p.n_tiles = r.n_tiles; p.tiles_per_chunk = r.tiles_per_chunk;
    conv3x3_wgrad_kernel<<<dim3(r.n_chunks, Cout / 64), THREADS, smem, st>>>(p);
    L3C_LAUNCH_CHECK("conv3x3_wgrad_kernel");
    const int n_out = Cout * NCOL + Cout;
    conv3x3_wgrad_finish_kernel<<<ceil_div(n_out, 256), 256, 0, st>>>(work_dev, r.n_chunks, Cout, dw_dev, db_dev);
    L3C_LAUNCH_CHECK("conv3x3_wgrad_finish_kernel");
    return L3C_OK;
}
