// bicubic.cu -- Pillow-compatible bicubic x0.5 down-sampling of uint8 planes (RGB baselines only).
//
// The reference's "encoder" for cr_rgb_shared.cf / cr_rgb.cf is PIL.Image.resize(.., BICUBIC) on the
// CPU (the reference's src/dataloaders/images_loader.py:277-293, called from modules/net.py:75).
// Pillow is a third-party, un-pinned dependency of the reference; this file restates the published
// algorithm of Pillow's two-pass resampler (src/libImaging/Resample.c: precompute_coeffs,
// normalize_coeffs_8bpc, ImagingResampleHorizontal_8bpc / Vertical_8bpc): separable, Keys cubic a=-0.5,
// support scaled by the down-scale factor, coefficients normalised then rounded to 22-bit fixed point,
// accumulation started at 2^21, arithmetic shift and clamp to [0,255], an 8-bit intermediate between the
// passes.  The horizontal pass runs first, except on images more than 100 times taller than wide
// (H > 100 * W), which Pillow 12 resizes vertically first.
//
// tests/test_bicubic_host.py pins an int64 restatement of that algorithm bit for bit to the installed
// Pillow (every H, W in 2..40, tall, flat and multi-megapixel shapes, content that drives both passes past
// both clamps) and shows that plausible mis-restatements differ from Pillow.  tests/test_gpu_bicubic.py
// checks this kernel bit for bit against both: the sweep, block edges of the x grid, batches, the grid
// limits below, large images, side streams, and every call the codec makes on every RGB-baseline path.
#include <math.h>

#include <vector>

#include "common.cuh"

namespace l3c {

constexpr int PRECISION_BITS = 32 - 8 - 2;

static double cubic_a05(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

// returns ksize; bounds[2*i] = first input index, bounds[2*i+1] = tap count; kk[i*ksize + t]
static int precompute(int in_size, int out_size, std::vector<int> &bounds, std::vector<int> &kk) {
    const double scale = (double)in_size / out_size;
    const double fscale = scale < 1.0 ? 1.0 : scale;
    const double support = 2.0 * fscale;
    const int ksize = (int)ceil(support) * 2 + 1;
    bounds.assign((size_t)out_size * 2, 0);
    kk.assign((size_t)out_size * ksize, 0);
    std::vector<double> k(ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        const double ss = 1.0 / fscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            k[x] = cubic_a05((x + xmin - center + 0.5) * ss);
            ww += k[x];
        }
        for (int x = 0; x < xmax; ++x) {
            double w = k[x];
            if (ww != 0.0) w /= ww;
            kk[(size_t)xx * ksize + x] = (w < 0) ? (int)(-0.5 + w * (1 << PRECISION_BITS))
                                                 : (int)(0.5 + w * (1 << PRECISION_BITS));
        }
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
    return ksize;
}

__device__ __forceinline__ uint8_t clip8(int v) {
    v >>= PRECISION_BITS;
    return (uint8_t)min(max(v, 0), 255);
}

// in: [planes][H][Win] -> out: [planes][H][Wout]
__global__ void resample_h_kernel(const uint8_t *__restrict__ in, int H, int Win, int Wout,
                                  const int *__restrict__ bounds, const int *__restrict__ kk, int ksize,
                                  uint8_t *__restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int pl = blockIdx.z;
    if (x >= Wout) return;
    const int x0 = bounds[2 * x], cnt = bounds[2 * x + 1];
    const uint8_t *row = in + ((size_t)pl * H + y) * Win;
    int ss = 1 << (PRECISION_BITS - 1);
    for (int t = 0; t < cnt; ++t) ss += (int)row[x0 + t] * kk[x * ksize + t];
    out[((size_t)pl * H + y) * Wout + x] = clip8(ss);
}

// in: [planes][Hin][W] -> out: [planes][Hout][W]
__global__ void resample_v_kernel(const uint8_t *__restrict__ in, int Hin, int Hout, int W,
                                  const int *__restrict__ bounds, const int *__restrict__ kk, int ksize,
                                  uint8_t *__restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    const int pl = blockIdx.z;
    if (x >= W) return;
    const int y0 = bounds[2 * y], cnt = bounds[2 * y + 1];
    int ss = 1 << (PRECISION_BITS - 1);
    for (int t = 0; t < cnt; ++t) ss += (int)in[((size_t)pl * Hin + y0 + t) * W + x] * kk[y * ksize + t];
    out[((size_t)pl * Hout + y) * W + x] = clip8(ss);
}

}  // namespace l3c

extern "C" int l3c_bicubic_half_u8(const uint8_t *in_dev, int N, int H, int W, uint8_t *out_dev,
                                   void *stream) {
    using namespace l3c;
    L3C_REQUIRE(in_dev && out_dev && N >= 1 && H >= 2 && W >= 2, "l3c_bicubic_half_u8: bad arguments");
    const int Ho = (int)(H * 0.5), Wo = (int)(W * 0.5);
    const int planes = N * 3;
    L3C_REQUIRE(planes <= 65535 && H <= 65535, "l3c_bicubic_half_u8: grid limits");
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int> bh, kh, bv, kv;
    const int ksh = precompute(W, Wo, bh, kh);
    const int ksv = precompute(H, Ho, bv, kv);
    int *d_bh, *d_kh, *d_bv, *d_kv;
    uint8_t *tmp;
    L3C_CUDA(cudaMallocAsync(&d_bh, bh.size() * 4, st));
    L3C_CUDA(cudaMallocAsync(&d_kh, kh.size() * 4, st));
    L3C_CUDA(cudaMallocAsync(&d_bv, bv.size() * 4, st));
    L3C_CUDA(cudaMallocAsync(&d_kv, kv.size() * 4, st));
    // Pillow 12's pass order: vertical first only for images more than 100x taller than wide
    const bool v_first = (long long)H > 100LL * W;
    L3C_CUDA(cudaMallocAsync(&tmp, (size_t)planes * (v_first ? (size_t)Ho * W : (size_t)H * Wo), st));
    L3C_CUDA(cudaMemcpyAsync(d_bh, bh.data(), bh.size() * 4, cudaMemcpyHostToDevice, st));
    L3C_CUDA(cudaMemcpyAsync(d_kh, kh.data(), kh.size() * 4, cudaMemcpyHostToDevice, st));
    L3C_CUDA(cudaMemcpyAsync(d_bv, bv.data(), bv.size() * 4, cudaMemcpyHostToDevice, st));
    L3C_CUDA(cudaMemcpyAsync(d_kv, kv.data(), kv.size() * 4, cudaMemcpyHostToDevice, st));
    // the pageable host vectors above are consumed synchronously by cudaMemcpyAsync (staged copy)
    if (v_first) {
        resample_v_kernel<<<dim3(ceil_div(W, 128), Ho, planes), 128, 0, st>>>(in_dev, H, Ho, W, d_bv, d_kv, ksv, tmp);
        L3C_LAUNCH_CHECK("resample_v_kernel");
        resample_h_kernel<<<dim3(ceil_div(Wo, 128), Ho, planes), 128, 0, st>>>(tmp, Ho, W, Wo, d_bh, d_kh, ksh, out_dev);
        L3C_LAUNCH_CHECK("resample_h_kernel");
    } else {
        resample_h_kernel<<<dim3(ceil_div(Wo, 128), H, planes), 128, 0, st>>>(in_dev, H, W, Wo, d_bh, d_kh, ksh, tmp);
        L3C_LAUNCH_CHECK("resample_h_kernel");
        resample_v_kernel<<<dim3(ceil_div(Wo, 128), Ho, planes), 128, 0, st>>>(tmp, H, Ho, Wo, d_bv, d_kv, ksv, out_dev);
        L3C_LAUNCH_CHECK("resample_v_kernel");
    }
    L3C_CUDA(cudaFreeAsync(d_bh, st));
    L3C_CUDA(cudaFreeAsync(d_kh, st));
    L3C_CUDA(cudaFreeAsync(d_bv, st));
    L3C_CUDA(cudaFreeAsync(d_kv, st));
    L3C_CUDA(cudaFreeAsync(tmp, st));
    return L3C_OK;
}
