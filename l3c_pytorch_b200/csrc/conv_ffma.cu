// conv_ffma.cu -- fp32 CUDA-core convolution (precision mode L3C_PREC_FP32) plus the small
// per-pixel layers of the L3C stack, NHWC.
//
// This is the bit-faithful fp32 path: every output element is accumulated in one fixed order
// (input-channel chunk -> filter tap -> channel), independent of batch size, image size or tile
// position, so the encoder's full forward pass and the decoder's three incremental get_P passes
// produce identical parameters (SURVEY.md section 7, "enc/dec bit-exactness").  The tensor-core
// kernels (conv_f16.cu, conv_tf32.cu, conv_f16x2.cu) keep the same property with a different, also fixed, order.
//
// Reference layers covered (all nn.Conv2d fp32 via cuDNN/MKL-DNN in the reference):
//   default_conv 3x3 / dilated 3x3 / 5x5 stride 2 / 1x1 ........ pytorch_ext.py:57-61
//   ResBlock conv-ReLU-conv, += x ................................ modules/edsr.py:63-89
//   Upsampler conv 64->256 + PixelShuffle(2) ...................... modules/edsr.py:92-119
//   MeanShift x2 (sub_rgb_mean, RGBHead) .......................... modules/edsr.py:52-60,
//                                                                  multiscale_network.py:181-183
//   to_q 1x1 + Quantizer (eval) ................................... modules/net.py:116-148,
//                                                                  modules/quantizer.py:62-90
#include <cuda_fp16.h>

#include "common.cuh"

namespace l3c {

// ------------------------------------------------------------------------------------------
// generic direct convolution: CTA = 8x16 output pixels x 64 output channels, 128 threads,
// thread = 8 pixels x 8 channels.  K loop = (chunk of 32 input channels) x (filter taps).
// ------------------------------------------------------------------------------------------
constexpr int TH = 8, TW = 16;
constexpr int CK = 32;            // input channels per chunk
constexpr int CKP = CK + 4;       // smem pixel pitch (floats): 16B aligned, bank-staggered
constexpr int CO_TILE = 64;
constexpr int CONV_THREADS = 128;

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ float round_tf32(float x) {      // round-to-nearest TF32 image of x
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// two floats -> packed fp16 pair (round-to-nearest-even, saturating): the F16 operand image (conv_f16.cu)
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
__device__ __forceinline__ void store_h(void *base, size_t idx, float v) {
    reinterpret_cast<uint16_t *>(base)[idx] = (uint16_t)(pack_h2(v, 0.f) & 0xFFFFu);
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
}

template <int KS, int S>
__global__ void __launch_bounds__(CONV_THREADS)
conv_ffma_kernel(l3c_conv_t p, int Ho, int Wo, int tiles_x, int pad) {
    extern __shared__ __align__(16) float smem[];
    const int D = p.dilation;
    const int HR = (TH - 1) * S + (KS - 1) * D + 1;
    const int HC = (TW - 1) * S + (KS - 1) * D + 1;
    float *halo = smem;                                  // [HR*HC][CKP]
    float *wbuf = smem + (size_t)HR * HC * CKP;          // [2][CK][CO_TILE]

    const int tid = threadIdx.x;
    const int tx = tid & 7;                              // channel group: co = 8*tx .. 8*tx+7
    const int ty = tid >> 3;                             // pixel group
    const int prow = ty >> 1;
    const int phalf = ty & 1;                            // columns 2*j + phalf
    const int n = blockIdx.z;
    const int ct = blockIdx.y;                           // output-channel tile
    const int oy0 = (blockIdx.x / tiles_x) * TH;
    const int ox0 = (blockIdx.x % tiles_x) * TW;
    const int iy0 = oy0 * S - pad;
    const int ix0 = ox0 * S - pad;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    const int nchunks = (p.Cin + CK - 1) / CK;
    const int T = nchunks * KS * KS;
    const float *xin = p.x + (size_t)n * p.H * p.W * p.x_pitch;

    auto issue_w = [&](int t) {
        const int chunk = t / (KS * KS), tap = t % (KS * KS);
        float *dst = wbuf + (size_t)(t & 1) * CK * CO_TILE;
        // 32 rows x 64 floats = 512 float4, 4 per thread
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int q = tid + i * CONV_THREADS;
            const int row = q >> 4, c4 = (q & 15) * 4;
            const int ci = chunk * CK + row;
            float *d = dst + row * CO_TILE + c4;
            if (ci < p.Cin) {
                cp_async16(d, p.w + ((size_t)tap * p.Cin + ci) * p.cout_pad + ct * CO_TILE + c4);
            } else {
                *reinterpret_cast<float4 *>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    };

    issue_w(0);
    for (int t = 0; t < T; ++t) {
        const int chunk = t / (KS * KS), tap = t % (KS * KS);
        if (tap == 0) {
            __syncthreads();                              // everyone is done with the old halo
            const int c0 = chunk * CK;
            const int npix = HR * HC;
            for (int q = tid; q < npix * (CK / 4); q += CONV_THREADS) {
                const int pix = q >> 3, c4 = (q & 7) * 4;
                const int iy = iy0 + pix / HC, ix = ix0 + pix % HC;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W && c0 + c4 + 4 <= p.x_pitch)
                    v = __ldg(reinterpret_cast<const float4 *>(
                        xin + ((size_t)iy * p.W + ix) * p.x_pitch + c0 + c4));
                *reinterpret_cast<float4 *>(halo + (size_t)pix * CKP + c4) = v;
            }
        }
        cp_async_wait_all();
        __syncthreads();
        if (t + 1 < T) issue_w(t + 1);

        const int ky = tap / KS, kx = tap % KS;
        const float *wb = wbuf + (size_t)(t & 1) * CK * CO_TILE + tx * 8;
        const float *hb = halo + ((size_t)(prow * S + ky * D) * HC + (phalf * S + kx * D)) * CKP;
#pragma unroll 2
        for (int k4 = 0; k4 < CK; k4 += 4) {
            float4 a[8];
#pragma unroll
            for (int j = 0; j < 8; ++j)
                a[j] = *reinterpret_cast<const float4 *>(hb + (size_t)(2 * j * S) * CKP + k4);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 b0 = *reinterpret_cast<const float4 *>(wb + (k4 + kk) * CO_TILE);
                const float4 b1 = *reinterpret_cast<const float4 *>(wb + (k4 + kk) * CO_TILE + 4);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float av = (kk == 0) ? a[j].x : (kk == 1) ? a[j].y : (kk == 2) ? a[j].z : a[j].w;
                    acc[j][0] = fmaf(av, b0.x, acc[j][0]);
                    acc[j][1] = fmaf(av, b0.y, acc[j][1]);
                    acc[j][2] = fmaf(av, b0.z, acc[j][2]);
                    acc[j][3] = fmaf(av, b0.w, acc[j][3]);
                    acc[j][4] = fmaf(av, b1.x, acc[j][4]);
                    acc[j][5] = fmaf(av, b1.y, acc[j][5]);
                    acc[j][6] = fmaf(av, b1.z, acc[j][6]);
                    acc[j][7] = fmaf(av, b1.w, acc[j][7]);
                }
            }
        }
    }

    // ---- epilogue: bias, ReLU, residual, store (plain / channel slice / pixel shuffle) ----
    const int co0 = ct * CO_TILE + tx * 8;
    if (co0 >= p.Cout) return;
    float bias[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) bias[c] = __ldg(p.bias + co0 + c);   // bias is padded to cout_pad
    const int oy = oy0 + prow;
    if (oy >= Ho) return;
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool shuffle = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
    const bool round_y = (p.flags & L3C_CONV_ROUND_TF32) != 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int ox = ox0 + 2 * j + phalf;
        if (ox >= Wo) continue;
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            v[c] = acc[j][c] + bias[c];
            if (relu) v[c] = fmaxf(v[c], 0.f);
        }
        if (!shuffle) {
            const size_t off = (((size_t)n * Ho + oy) * Wo + ox) * p.y_pitch + p.y_coff + co0;
            const bool vec = ((p.y_pitch | p.y_coff) & 3) == 0 && co0 + 8 <= p.Cout;
            if (vec) {
                if (p.residual) {
                    const float4 r0 = __ldg(reinterpret_cast<const float4 *>(p.residual + off));
                    const float4 r1 = __ldg(reinterpret_cast<const float4 *>(p.residual + off + 4));
                    v[0] += r0.x; v[1] += r0.y; v[2] += r0.z; v[3] += r0.w;
                    v[4] += r1.x; v[5] += r1.y; v[6] += r1.z; v[7] += r1.w;
                }
                if (p.y_tf32) {
                    *reinterpret_cast<float4 *>(p.y_tf32 + off) =
                        make_float4(round_tf32(v[0]), round_tf32(v[1]), round_tf32(v[2]), round_tf32(v[3]));
                    *reinterpret_cast<float4 *>(p.y_tf32 + off + 4) =
                        make_float4(round_tf32(v[4]), round_tf32(v[5]), round_tf32(v[6]), round_tf32(v[7]));
                }
                if (p.y_h && ((p.y_pitch | p.y_coff) & 7) == 0) {
                    *reinterpret_cast<uint4 *>(reinterpret_cast<uint16_t *>(p.y_h) + off) =
                        make_uint4(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]), pack_h2(v[4], v[5]), pack_h2(v[6], v[7]));
                } else if (p.y_h) {
#pragma unroll
                    for (int c = 0; c < 8; ++c) store_h(p.y_h, off + c, v[c]);
                }
                if (round_y) {
#pragma unroll
                    for (int c = 0; c < 8; ++c) v[c] = round_tf32(v[c]);
                }
                *reinterpret_cast<float4 *>(p.y + off) = make_float4(v[0], v[1], v[2], v[3]);
                *reinterpret_cast<float4 *>(p.y + off + 4) = make_float4(v[4], v[5], v[6], v[7]);
            } else {
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    if (co0 + c < p.Cout) {
                        float o = v[c];
                        if (p.residual) o += __ldg(p.residual + off + c);
                        if (p.y_tf32) p.y_tf32[off + c] = round_tf32(o);
                        if (p.y_h) store_h(p.y_h, off + c, o);
                        p.y[off + c] = round_y ? round_tf32(o) : o;
                    }
                }
            }
        } else {
            // out[n, 2*oy+i, 2*ox+jj, cq] = y[n, oy, ox, 4*cq + 2*i + jj];  pitch = y_pitch
            const int Ho2 = Ho * 2, Wo2 = Wo * 2;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int co = co0 + c;
                if (co >= p.Cout) continue;
                const int cq = co >> 2, i = (co >> 1) & 1, jj = co & 1;
                const size_t off = (((size_t)n * Ho2 + 2 * oy + i) * Wo2 + 2 * ox + jj) * p.y_pitch +
                                   p.y_coff + cq;
                float o = v[c];
                if (p.residual) o += __ldg(p.residual + off);
                if (p.y_tf32) p.y_tf32[off] = round_tf32(o);
                if (p.y_h) store_h(p.y_h, off, o);
                p.y[off] = round_y ? round_tf32(o) : o;
            }
        }
    }
}

template <int KS, int S>
static int launch_conv(const l3c_conv_t &p, int Ho, int Wo, int pad, cudaStream_t st) {
    const int D = p.dilation;
    const int HR = (TH - 1) * S + (KS - 1) * D + 1;
    const int HC = (TW - 1) * S + (KS - 1) * D + 1;
    const size_t smem = ((size_t)HR * HC * CKP + 2 * CK * CO_TILE) * sizeof(float);
    L3C_REQUIRE(smem <= 227 * 1024, "l3c_conv2d: tile needs %zu B of shared memory", smem);
    auto kern = conv_ffma_kernel<KS, S>;
    static size_t configured_dev[64] = {};   // per (KS,S) instantiation and device
    size_t &configured = configured_dev[current_device_slot()];
    if (smem > configured) {
        L3C_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    const int tiles_x = ceil_div(Wo, TW), tiles_y = ceil_div(Ho, TH);
    dim3 grid(tiles_x * tiles_y, ceil_div(p.Cout, CO_TILE), p.N);
    kern<<<grid, CONV_THREADS, smem, st>>>(p, Ho, Wo, tiles_x, pad);
    L3C_LAUNCH_CHECK("conv_ffma_kernel");
    return L3C_OK;
}

int conv2d_ffma(const l3c_conv_t &p, cudaStream_t st) {
    const int pad = (p.dilation == 1) ? p.ksize / 2 : p.dilation;      // pytorch_ext.py:58
    const int Ho = (p.H + 2 * pad - p.dilation * (p.ksize - 1) - 1) / p.stride + 1;
    const int Wo = (p.W + 2 * pad - p.dilation * (p.ksize - 1) - 1) / p.stride + 1;
    if (p.ksize == 3 && p.stride == 1) return launch_conv<3, 1>(p, Ho, Wo, pad, st);
    if (p.ksize == 1 && p.stride == 1) return launch_conv<1, 1>(p, Ho, Wo, pad, st);
    if (p.ksize == 5 && p.stride == 2) return launch_conv<5, 2>(p, Ho, Wo, pad, st);
    set_error("l3c_conv2d: unsupported ksize=%d stride=%d (L3C uses 3x3/s1, 1x1/s1, 5x5/s2)",
              p.ksize, p.stride);
    return L3C_EINVAL;
}

// ------------------------------------------------------------------------------------------
// per-pixel layers
// ------------------------------------------------------------------------------------------
__global__ void rgb_prep_kernel(const uint8_t *__restrict__ img, const float *__restrict__ A1,
                                const float *__restrict__ b1, const float *__restrict__ A2,
                                const float *__restrict__ b2, int HW, float *__restrict__ xsub,
                                float *__restrict__ t) {
    const int n = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    float x[3], y[3], z[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = (float)img[((size_t)n * 3 + c) * HW + p];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < 3; ++j) a = fmaf(A1[c * 3 + j], x[j], a);
        y[c] = a + b1[c];
    }
    if (xsub) {
#pragma unroll
        for (int c = 0; c < 3; ++c) xsub[((size_t)n * HW + p) * 3 + c] = y[c];
    }
    if (t) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < 3; ++j) a = fmaf(A2[c * 3 + j], y[j], a);
            z[c] = a + b2[c];
        }
        *reinterpret_cast<float4 *>(t + ((size_t)n * HW + p) * 4) = make_float4(z[0], z[1], z[2], 0.f);
    }
}

// RGB head for the F16 tensor-core path: the two MeanShift affines (as rgb_prep_kernel) followed by an im2col of
// the 3x3 neighbourhood -- per pixel one 128-byte row of 64 FP16 values, element tap*3 + c = normalised channel c
// of the pixel at tap (ky, kx) (0 outside the image: the conv's zero padding acts on the NORMALISED input,
// head.py:31-59), elements 27..63 zero.  The 3 -> 64 conv then is a 1x1 GEMM with K = 64 on the tensor cores
// (conv1x1_f16_kernel) instead of 3.2 ms of CUDA-core work per 16 x 512^2 batch.
__global__ void rgb_im2col_kernel(const uint8_t *__restrict__ img, const float *__restrict__ A1,
                                  const float *__restrict__ b1, const float *__restrict__ A2,
                                  const float *__restrict__ b2, int H, int W, const int *__restrict__ ext,
                                  uint4 *__restrict__ out) {
    const int n = blockIdx.y;
    const int HW = H * W;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const int y0 = p / W, x0 = p % W;
    // ragged batch: image n is [0,Hn) x [0,Wn) of the padded tensor, and its zero padding starts there
    const int Hn = ext ? ext[2 * n] : H, Wn = ext ? ext[2 * n + 1] : W;
    float v[28];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int yy = y0 + tap / 3 - 1, xx = x0 + tap % 3 - 1;
        const bool in = yy >= 0 && yy < Hn && xx >= 0 && xx < Wn;
        float x[3], y[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) x[c] = in ? (float)img[((size_t)n * 3 + c) * HW + yy * W + xx] : 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < 3; ++j) a = fmaf(A1[c * 3 + j], x[j], a);
            y[c] = a + b1[c];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < 3; ++j) a = fmaf(A2[c * 3 + j], y[j], a);
            v[tap * 3 + c] = in ? a + b2[c] : 0.f;
        }
    }
    v[27] = 0.f;
    uint4 *dst = out + ((size_t)n * HW + p) * 8;            // 8 x 16 bytes
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = q * 8 + 2 * i;
            w[i] = (e < 28) ? pack_h2(v[e], v[e + 1]) : 0u;
        }
        dst[q] = make_uint4(w[0], w[1], w[2], w[3]);
    }
#pragma unroll
    for (int q = 4; q < 8; ++q) dst[q] = make_uint4(0u, 0u, 0u, 0u);
}

// to_q (1x1, Cf -> C) + hard quantiser.  One thread per pixel; C <= 8.
constexpr int QMAXC = 8;
__global__ void quantize_head_kernel(const float *__restrict__ f, const float *__restrict__ w,
                                     const float *__restrict__ bias,
                                     const float *__restrict__ levels, int HW, int Cf, int C, int L,
                                     uint8_t *__restrict__ sym, float *__restrict__ bnq,
                                     int bnq_pitch) {
    extern __shared__ float sw[];          // [Cf][C] weights, then [L] levels
    float *slev = sw + Cf * C;
    for (int i = threadIdx.x; i < Cf * C; i += blockDim.x) sw[i] = w[i];
    for (int i = threadIdx.x; i < L; i += blockDim.x) slev[i] = levels[i];
    __syncthreads();
    const int n = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    float q[QMAXC];
#pragma unroll
    for (int c = 0; c < QMAXC; ++c) q[c] = 0.f;
    const float4 *fp = reinterpret_cast<const float4 *>(f + ((size_t)n * HW + p) * Cf);
    for (int k4 = 0; k4 < Cf / 4; ++k4) {
        const float4 v = __ldg(fp + k4);
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int c = 0; c < QMAXC; ++c)
                if (c < C) q[c] = fmaf(vv[kk], sw[(k4 * 4 + kk) * C + c], q[c]);
    }
#pragma unroll
    for (int c = 0; c < QMAXC; ++c) {
        if (c >= C) {
            if (c < bnq_pitch) bnq[((size_t)n * HW + p) * bnq_pitch + c] = 0.f;
            continue;
        }
        const float x = q[c] + bias[c];
        int best = 0;
        float bd = (x - slev[0]) * (x - slev[0]);
        for (int l = 1; l < L; ++l) {
            const float d = (x - slev[l]) * (x - slev[l]);
            if (d < bd) {                    // strict: first minimum wins, as torch.min does
                bd = d;
                best = l;
            }
        }
        sym[((size_t)n * C + c) * HW + p] = (uint8_t)best;
        bnq[((size_t)n * HW + p) * bnq_pitch + c] = slev[best];
    }
}

__global__ void symbols_to_values_kernel(const uint8_t *__restrict__ sym,
                                         const float *__restrict__ values,
                                         const float *__restrict__ shift, int HW, int C, int pitch,
                                         float *__restrict__ out) {
    const int n = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    for (int c = 0; c < pitch; ++c) {
        float v = 0.f;
        if (c < C) {
            v = __ldg(values + sym[((size_t)n * C + c) * HW + p]);
            if (shift) v -= __ldg(shift + c);
        }
        out[((size_t)n * HW + p) * pitch + c] = v;
    }
}

}  // namespace l3c

extern "C" int l3c_rgb_prep(const uint8_t *img_dev, const float *A1, const float *b1,
                            const float *A2, const float *b2, int N, int HW, float *xsub_dev,
                            float *t_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(img_dev && A1 && b1 && N >= 1 && HW >= 1 && N <= 65535, "l3c_rgb_prep: bad arguments");
    L3C_REQUIRE(!t_dev || (A2 && b2), "l3c_rgb_prep: second affine missing");
    dim3 grid(ceil_div(HW, 256), N);
    rgb_prep_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(img_dev, A1, b1, A2, b2, HW, xsub_dev, t_dev);
    L3C_LAUNCH_CHECK("rgb_prep_kernel");
    return L3C_OK;
}

extern "C" int l3c_rgb_im2col_f16_ragged(const uint8_t *img_dev, const float *A1, const float *b1, const float *A2,
                                         const float *b2, int N, int H, int W, const int *extents_dev, void *out_h_dev,
                                         void *stream) {
    using namespace l3c;
    L3C_REQUIRE(img_dev && A1 && b1 && A2 && b2 && out_h_dev && N >= 1 && H >= 1 && W >= 1 && N <= 65535,
                "l3c_rgb_im2col_f16: bad arguments");
    dim3 grid(ceil_div(H * W, 128), N);
    rgb_im2col_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(img_dev, A1, b1, A2, b2, H, W, extents_dev,
                                                              reinterpret_cast<uint4 *>(out_h_dev));
    L3C_LAUNCH_CHECK("rgb_im2col_kernel");
    return L3C_OK;
}

extern "C" int l3c_rgb_im2col_f16(const uint8_t *img_dev, const float *A1, const float *b1, const float *A2,
                                  const float *b2, int N, int H, int W, void *out_h_dev, void *stream) {
    return l3c_rgb_im2col_f16_ragged(img_dev, A1, b1, A2, b2, N, H, W, nullptr, out_h_dev, stream);
}

extern "C" int l3c_quantize_head(const float *f_dev, const float *w_dev, const float *bias_dev,
                                 const float *levels_dev, int N, int HW, int Cf, int C, int L,
                                 uint8_t *sym_dev, float *bnq_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(f_dev && w_dev && bias_dev && levels_dev && sym_dev && bnq_dev, "l3c_quantize_head: null pointer");
    L3C_REQUIRE(C >= 1 && C <= QMAXC && Cf % 4 == 0 && L >= 1 && L <= 256 && N >= 1 && N <= 65535,
                "l3c_quantize_head: C=%d Cf=%d L=%d N=%d", C, Cf, L, N);
    dim3 grid(ceil_div(HW, 128), N);
    const size_t smem = (size_t)(Cf * C + L) * sizeof(float);
    quantize_head_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>(
        f_dev, w_dev, bias_dev, levels_dev, HW, Cf, C, L, sym_dev, bnq_dev, 8);
    L3C_LAUNCH_CHECK("quantize_head_kernel");
    return L3C_OK;
}

extern "C" int l3c_symbols_to_values(const uint8_t *sym_dev, const float *values_dev,
                                     const float *shift_dev, int N, int HW, int C, int L,
                                     float *out_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(sym_dev && values_dev && out_dev && C >= 1 && C <= 8 && N >= 1 && N <= 65535 && L >= 1,
                "l3c_symbols_to_values: bad arguments");
    dim3 grid(ceil_div(HW, 256), N);
    symbols_to_values_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(sym_dev, values_dev, shift_dev,
                                                                     HW, C, 8, out_dev);
    L3C_LAUNCH_CHECK("symbols_to_values_kernel");
    return L3C_OK;
}
