// capi.cu -- error plumbing, dispatch and the five drop-in exports of the reference's native module
// (torchac_backend_{cpu,gpu}: /root/reference/src/torchac/torchac_backend/torchac.cpp:433-443),
// implemented on top of the batched kernels of range_coder.cu / dmll.cu.
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "dmll_math.cuh"

namespace l3c {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---- launch log: every kernel launch of this library is counted under its kernel name --------
namespace {
struct LaunchEntry {
    const char *name;      // string literal at the launch site
    unsigned long long n;
};
constexpr int MAX_LOG = 64;
LaunchEntry g_log[MAX_LOG];
int g_log_n = 0;
std::mutex g_log_mu;
}  // namespace

void count_launch(const char *kernel_name) {
    std::lock_guard<std::mutex> lk(g_log_mu);
    for (int i = 0; i < g_log_n; ++i) {
        if (g_log[i].name == kernel_name || strcmp(g_log[i].name, kernel_name) == 0) {
            g_log[i].n++;
            return;
        }
    }
    if (g_log_n < MAX_LOG) g_log[g_log_n++] = LaunchEntry{kernel_name, 1ull};
}

int sm_count() {
    static int counts[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!counts[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        counts[dev] = n;
    }
    return counts[dev];
}

int conv2d_ffma(const l3c_conv_t &p, cudaStream_t st);
int conv2d_tf32(const l3c_conv_t &p, cudaStream_t st);
int conv2d_f16(const l3c_conv_t &p, cudaStream_t st);
int conv2d_f16x2(const l3c_conv_t &p, cudaStream_t st);

// ---- helper kernels for the single-stream (reference-shaped) API -----------------------------

// intervals from an explicit table: torchac.cpp:178-182
__global__ void table_intervals_kernel(const uint16_t *__restrict__ cdf, const int16_t *__restrict__ sym,
                                       int64_t n_sym, int Lp, uint32_t *__restrict__ iv) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sym) return;
    const int s = sym[i];
    const uint32_t lo = cdf[i * Lp + s];
    const uint32_t hi = (s == Lp - 2) ? 0x10000u : (uint32_t)cdf[i * Lp + s + 1];
    iv[i] = lo | ((hi - 1u) << 16);
}

// [n][Lp] rows -> [n][pitch] rows (the dead (L+1)-th entry is dropped, the tail is padding)
__global__ void repitch_kernel(const uint16_t *__restrict__ cdf, int64_t n_sym, int Lp, int pitch,
                               uint16_t *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sym * pitch) return;
    const int64_t r = i / pitch;
    const int e = (int)(i % pitch);
    out[i] = (e < Lp - 1) ? cdf[r * Lp + e] : (uint16_t)0;
}

// cdf[n][l] of torchac_kernel.cu:58-75 from [K][N] planes: dmll_math.cuh, plane_cdf_u16
__global__ void plane_intervals_kernel(const float *__restrict__ targets, const float *__restrict__ means,
                                       const float *__restrict__ log_scales,
                                       const float *__restrict__ probs, int K, int64_t N, int Lp,
                                       const int16_t *__restrict__ sym, uint32_t *__restrict__ iv) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int s = sym[n];
    const float scale = (float)(65536 - (Lp - 1));
    const uint32_t lo = plane_cdf_u16(means, log_scales, probs, K, N, n, targets[s], scale, s);
    const uint32_t hi = (s == Lp - 2) ? 0x10000u
                                      : plane_cdf_u16(means, log_scales, probs, K, N, n,
                                                      targets[s + 1], scale, s + 1);
    iv[n] = lo | ((hi - 1u) << 16);
}

__global__ void plane_table_kernel(const float *__restrict__ targets, const float *__restrict__ means,
                                   const float *__restrict__ log_scales,
                                   const float *__restrict__ probs, int K, int64_t N, int Lp, int pitch,
                                   uint16_t *__restrict__ table) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * pitch) return;
    const int64_t n = i / pitch;
    const int l = (int)(i % pitch);
    uint32_t v = 0;
    if (l < Lp - 1)
        v = plane_cdf_u16(means, log_scales, probs, K, N, n, targets[l], (float)(65536 - (Lp - 1)), l);
    table[i] = (uint16_t)v;
}

struct DevBuf {
    void *p = nullptr;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    int alloc(size_t bytes) {
        L3C_CUDA(cudaMalloc(&p, bytes ? bytes : 4));
        return L3C_OK;
    }
    template <typename T>
    T *as() { return reinterpret_cast<T *>(p); }
};

static int run_encode(const uint32_t *iv_dev, int64_t n_sym, uint8_t *out_host, size_t out_cap,
                      size_t *out_len) {
    // the slot bound (17 bits per symbol + the terminator), clamped to the largest uint32 multiple of 4: above it
    // the coder's saturated length exceeds the slot and the call fails instead of wrapping
    const size_t cap = std::min<size_t>((((size_t)n_sym * 17 + 7) / 8 + 64 + 3) & ~(size_t)3, 0xFFFFFFFCu);
    DevBuf out, desc, len;
    if (int e = out.alloc(cap)) return e;
    if (int e = desc.alloc(sizeof(l3c_enc_stream_t))) return e;
    if (int e = len.alloc(4)) return e;
    l3c_enc_stream_t d;
    d.intervals = iv_dev;
    d.out = out.as<uint8_t>();
    d.n_sym = (uint32_t)n_sym;
    d.out_cap = (uint32_t)cap;
    L3C_CUDA(cudaMemcpy(desc.p, &d, sizeof(d), cudaMemcpyHostToDevice));
    if (int e = l3c_ac_encode_streams(desc.as<l3c_enc_stream_t>(), 1, len.as<uint32_t>(), nullptr)) return e;
    uint32_t n = 0;
    L3C_CUDA(cudaMemcpy(&n, len.p, 4, cudaMemcpyDeviceToHost));
    *out_len = n;
    if (n > out_cap || n > cap) {
        set_error("encode: %u bytes do not fit the %zu byte output buffer", n, out_cap);
        return L3C_EOVERFLOW;
    }
    L3C_CUDA(cudaMemcpy(out_host, out.p, n, cudaMemcpyDeviceToHost));
    return L3C_OK;
}

static int run_decode(const uint16_t *table_dev, int pitch, int64_t n_sym, int L,
                      const uint8_t *in_host, size_t in_len, int16_t *sym_out_host) {
    const size_t padded = ((in_len + 3) & ~(size_t)3) + 8;
    const size_t sym_bytes = (L > 256) ? 2 : 1;        // the decoder writes uint16 symbols for L > 256
    DevBuf in, sym, desc;
    if (int e = in.alloc(padded)) return e;
    if (int e = sym.alloc((size_t)n_sym * sym_bytes)) return e;
    if (int e = desc.alloc(sizeof(l3c_dec_stream_t))) return e;
    L3C_CUDA(cudaMemset(in.p, 0, padded));
    if (in_len) L3C_CUDA(cudaMemcpy(in.p, in_host, in_len, cudaMemcpyHostToDevice));
    l3c_dec_stream_t d;
    d.table = table_dev;
    d.in = in.as<uint8_t>();
    d.sym_out = sym.as<uint8_t>();
    d.state = nullptr;
    d.row_pitch = pitch;
    d.n_sym = (uint32_t)n_sym;
    d.in_len = (uint32_t)in_len;
    L3C_CUDA(cudaMemcpy(desc.p, &d, sizeof(d), cudaMemcpyHostToDevice));
    if (int e = l3c_ac_decode_streams(desc.as<l3c_dec_stream_t>(), 1, L, 0, (uint32_t)n_sym, nullptr)) return e;
    if (sym_bytes == 2) {
        L3C_CUDA(cudaMemcpy(sym_out_host, sym.p, (size_t)n_sym * 2, cudaMemcpyDeviceToHost));
        return L3C_OK;
    }
    std::vector<uint8_t> tmp((size_t)n_sym);
    L3C_CUDA(cudaMemcpy(tmp.data(), sym.p, (size_t)n_sym, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n_sym; ++i) sym_out_host[i] = (int16_t)tmp[(size_t)i];
    return L3C_OK;
}

// Lp <= 32769: the reference passes symbols as int16, so L = 32768 is the largest alphabet it can code
static int check_stream_args(const char *fn, int64_t n_sym, int Lp) {
    L3C_REQUIRE(n_sym >= 1 && n_sym < (1ll << 31), "%s: n_sym=%lld", fn, (long long)n_sym);
    L3C_REQUIRE(Lp >= 2 && Lp <= 32769, "%s: Lp=%d not in [2,32769]", fn, Lp);
    return L3C_OK;
}

}  // namespace l3c

using namespace l3c;

extern "C" const char *l3c_last_error(void) { return g_err; }
extern "C" int l3c_version(void) { return 100; }

extern "C" int l3c_cuda_supported(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return 0;
    }
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
    return major == 9 ? 1 : 0;
}

extern "C" int l3c_conv2d(const l3c_conv_t *p, void *stream) {
    L3C_REQUIRE(p && p->bias, "l3c_conv2d: null pointer");
    L3C_REQUIRE(p->precision >= L3C_PREC_FP32 && p->precision <= L3C_PREC_F16X2, "l3c_conv2d: unknown precision %d", p->precision);
    if (p->precision == L3C_PREC_F16 || p->precision == L3C_PREC_F16X2) {
        L3C_REQUIRE(p->x_h && p->w_h && (p->y || p->y_h), "l3c_conv2d: F16 modes need x_h, w_h and y or y_h");
    } else {
        L3C_REQUIRE(p->x && p->w && p->y, "l3c_conv2d: null pointer");
    }
    L3C_REQUIRE(p->N >= 1 && p->N <= 65535 && p->H >= 1 && p->W >= 1, "l3c_conv2d: N=%d H=%d W=%d", p->N, p->H, p->W);
    L3C_REQUIRE(p->Cin >= 1 && p->x_pitch >= p->Cin && p->x_pitch % 4 == 0,
                "l3c_conv2d: Cin=%d x_pitch=%d (pitch must be a multiple of 4)", p->Cin, p->x_pitch);
    L3C_REQUIRE(p->Cout >= 1 && p->cout_pad >= p->Cout && p->cout_pad % 64 == 0,
                "l3c_conv2d: Cout=%d cout_pad=%d (must be padded to a multiple of 64)", p->Cout, p->cout_pad);
    L3C_REQUIRE(p->dilation >= 1 && (p->dilation == 1 || p->ksize == 3), "l3c_conv2d: dilation=%d ksize=%d", p->dilation, p->ksize);
    if (p->flags & L3C_CONV_PIXEL_SHUFFLE2) {
        L3C_REQUIRE(p->Cout % 4 == 0 && p->y_pitch >= p->y_coff + p->Cout / 4, "l3c_conv2d: pixel-shuffle pitch");
    } else {
        L3C_REQUIRE(p->y_pitch >= p->y_coff + p->Cout, "l3c_conv2d: y_pitch=%d y_coff=%d Cout=%d", p->y_pitch, p->y_coff, p->Cout);
    }
    if (p->precision == L3C_PREC_FP32) return conv2d_ffma(*p, (cudaStream_t)stream);
    if (p->precision == L3C_PREC_F16) return conv2d_f16(*p, (cudaStream_t)stream);
    if (p->precision == L3C_PREC_F16X2) return conv2d_f16x2(*p, (cudaStream_t)stream);
    return conv2d_tf32(*p, (cudaStream_t)stream);
}

extern "C" int l3c_encode_cdf(const uint16_t *cdf_host, int64_t n_sym, int Lp,
                              const int16_t *sym_host, uint8_t *out_host, size_t out_cap,
                              size_t *out_len) {
    if (int e = check_stream_args("l3c_encode_cdf", n_sym, Lp)) return e;
    L3C_REQUIRE(cdf_host && sym_host && out_host && out_len, "l3c_encode_cdf: null pointer");
    for (int64_t i = 0; i < n_sym; ++i)
        L3C_REQUIRE(sym_host[i] >= 0 && sym_host[i] <= Lp - 2, "l3c_encode_cdf: symbol %d at %lld outside [0,%d]",
                    (int)sym_host[i], (long long)i, Lp - 2);
    DevBuf cdf, sym, iv;
    if (int e = cdf.alloc((size_t)n_sym * Lp * 2)) return e;
    if (int e = sym.alloc((size_t)n_sym * 2)) return e;
    if (int e = iv.alloc((size_t)n_sym * 4)) return e;
    L3C_CUDA(cudaMemcpy(cdf.p, cdf_host, (size_t)n_sym * Lp * 2, cudaMemcpyHostToDevice));
    L3C_CUDA(cudaMemcpy(sym.p, sym_host, (size_t)n_sym * 2, cudaMemcpyHostToDevice));
    table_intervals_kernel<<<(unsigned)ceil_div64(n_sym, 256), 256>>>(cdf.as<uint16_t>(), sym.as<int16_t>(),
                                                                      n_sym, Lp, iv.as<uint32_t>());
    L3C_LAUNCH_CHECK("table_intervals_kernel");
    return run_encode(iv.as<uint32_t>(), n_sym, out_host, out_cap, out_len);
}

extern "C" int l3c_decode_cdf(const uint16_t *cdf_host, int64_t n_sym, int Lp, const uint8_t *in_host,
                              size_t in_len, int16_t *sym_out_host) {
    if (int e = check_stream_args("l3c_decode_cdf", n_sym, Lp)) return e;
    L3C_REQUIRE(cdf_host && sym_out_host && (in_host || in_len == 0), "l3c_decode_cdf: null pointer");
    const int L = Lp - 1;
    const int pitch = decode_pitch(L);
    DevBuf cdf, table;
    if (int e = cdf.alloc((size_t)n_sym * Lp * 2)) return e;
    if (int e = table.alloc((size_t)n_sym * pitch * 2)) return e;
    L3C_CUDA(cudaMemcpy(cdf.p, cdf_host, (size_t)n_sym * Lp * 2, cudaMemcpyHostToDevice));
    repitch_kernel<<<(unsigned)ceil_div64(n_sym * pitch, 256), 256>>>(cdf.as<uint16_t>(), n_sym, Lp, pitch,
                                                                      table.as<uint16_t>());
    L3C_LAUNCH_CHECK("repitch_kernel");
    return run_decode(table.as<uint16_t>(), pitch, n_sym, L, in_host, in_len, sym_out_host);
}

extern "C" int l3c_encode_logistic_mixture(const float *targets_dev, const float *means_dev,
                                           const float *log_scales_dev, const float *probs_dev, int K,
                                           int64_t n_sym, int Lp, const int16_t *sym_host,
                                           uint8_t *out_host, size_t out_cap, size_t *out_len) {
    if (int e = check_stream_args("l3c_encode_logistic_mixture", n_sym, Lp)) return e;
    L3C_REQUIRE(targets_dev && means_dev && log_scales_dev && probs_dev && sym_host && out_host && out_len && K >= 1,
                "l3c_encode_logistic_mixture: bad arguments");
    for (int64_t i = 0; i < n_sym; ++i)
        L3C_REQUIRE(sym_host[i] >= 0 && sym_host[i] <= Lp - 2, "l3c_encode_logistic_mixture: symbol out of range");
    DevBuf sym, iv;
    if (int e = sym.alloc((size_t)n_sym * 2)) return e;
    if (int e = iv.alloc((size_t)n_sym * 4)) return e;
    L3C_CUDA(cudaMemcpy(sym.p, sym_host, (size_t)n_sym * 2, cudaMemcpyHostToDevice));
    plane_intervals_kernel<<<(unsigned)ceil_div64(n_sym, 128), 128>>>(
        targets_dev, means_dev, log_scales_dev, probs_dev, K, n_sym, Lp, sym.as<int16_t>(), iv.as<uint32_t>());
    L3C_LAUNCH_CHECK("plane_intervals_kernel");
    return run_encode(iv.as<uint32_t>(), n_sym, out_host, out_cap, out_len);
}

extern "C" int l3c_decode_logistic_mixture(const float *targets_dev, const float *means_dev,
                                           const float *log_scales_dev, const float *probs_dev, int K,
                                           int64_t n_sym, int Lp, const uint8_t *in_host, size_t in_len,
                                           int16_t *sym_out_host) {
    if (int e = check_stream_args("l3c_decode_logistic_mixture", n_sym, Lp)) return e;
    L3C_REQUIRE(targets_dev && means_dev && log_scales_dev && probs_dev && sym_out_host && K >= 1 &&
                    (in_host || in_len == 0),
                "l3c_decode_logistic_mixture: bad arguments");
    const int L = Lp - 1;
    const int pitch = decode_pitch(L);
    DevBuf table;
    if (int e = table.alloc((size_t)n_sym * pitch * 2)) return e;
    plane_table_kernel<<<(unsigned)ceil_div64(n_sym * pitch, 256), 256>>>(
        targets_dev, means_dev, log_scales_dev, probs_dev, K, n_sym, Lp, pitch, table.as<uint16_t>());
    L3C_LAUNCH_CHECK("plane_table_kernel");
    return run_decode(table.as<uint16_t>(), pitch, n_sym, L, in_host, in_len, sym_out_host);
}

// launch log: "kernel_name count\n" per kernel launched since the last reset; returns the total number of
// launches (the text is truncated to `cap`, the return value is not).  reset != 0 clears the counters.
extern "C" long long l3c_launch_log(char *buf, size_t cap, int reset) {
    using namespace l3c;
    std::lock_guard<std::mutex> lk(g_log_mu);
    long long total = 0;
    size_t pos = 0;
    if (buf && cap) buf[0] = 0;
    for (int i = 0; i < g_log_n; ++i) {
        total += (long long)g_log[i].n;
        if (buf && pos + 1 < cap) {
            const int w = snprintf(buf + pos, cap - pos, "%s %llu\n", g_log[i].name, g_log[i].n);
            if (w > 0) pos += (size_t)w < cap - pos ? (size_t)w : cap - pos - 1;
        }
    }
    if (reset) g_log_n = 0;
    return total;
}

// ---- CTA trace of the persistent tensor-core kernels (L3C_CTA_TRACE builds) ----------------
#ifdef L3C_CTA_TRACE
namespace l3c {
namespace {
struct TraceLaunch {
    const char *name;
    unsigned gx, gy;
    long long first;
    cudaStream_t st;
};
std::mutex g_trace_mu;
l3c_cta_record_t *g_trace_rec = nullptr;
long long g_trace_cap = 0, g_trace_used = 0;
std::vector<TraceLaunch> g_trace_launches;
}  // namespace

CtaTraceArg cta_trace_launch(const char *name, dim3 grid, cudaStream_t st) {
    std::lock_guard<std::mutex> lk(g_trace_mu);
    const long long n = (long long)grid.x * grid.y;
    if (!g_trace_rec || g_trace_used + n > g_trace_cap) return CtaTraceArg{nullptr, -1};
    const CtaTraceArg a{g_trace_rec + g_trace_used, (int)g_trace_launches.size()};
    g_trace_launches.push_back(TraceLaunch{name, grid.x, grid.y, g_trace_used, st});
    g_trace_used += n;
    return a;
}
}  // namespace l3c
#endif

extern "C" int l3c_cta_trace_register(l3c_cta_record_t *records_dev, int64_t capacity) {
    using namespace l3c;
#ifdef L3C_CTA_TRACE
    L3C_REQUIRE(capacity >= 0, "l3c_cta_trace_register: capacity %lld", (long long)capacity);
    std::lock_guard<std::mutex> lk(g_trace_mu);
    g_trace_rec = records_dev;
    g_trace_cap = records_dev ? capacity : 0;
    g_trace_used = 0;
    g_trace_launches.clear();
    return L3C_OK;
#else
    (void)records_dev; (void)capacity;
    set_error("l3c_cta_trace_register: this library is built without L3C_CTA_TRACE");
    return L3C_EUNSUPPORTED;
#endif
}

extern "C" int l3c_cta_trace_launches(char *buf, size_t cap, int64_t *n_records) {
    using namespace l3c;
#ifdef L3C_CTA_TRACE
    std::lock_guard<std::mutex> lk(g_trace_mu);
    size_t pos = 0;
    if (buf && cap) buf[0] = 0;
    for (size_t i = 0; i < g_trace_launches.size(); ++i) {
        const TraceLaunch &l = g_trace_launches[i];
        if (buf && pos + 1 < cap) {
            const int w = snprintf(buf + pos, cap - pos, "%zu %s %u %u %lld %p\n", i, l.name, l.gx, l.gy, l.first,
                                   (void *)l.st);
            if (w > 0) pos += (size_t)w < cap - pos ? (size_t)w : cap - pos - 1;
        }
    }
    if (n_records) *n_records = g_trace_used;
    return L3C_OK;
#else
    (void)buf; (void)cap; (void)n_records;
    set_error("l3c_cta_trace_launches: this library is built without L3C_CTA_TRACE");
    return L3C_EUNSUPPORTED;
#endif
}

// ---------------------------------------------------------------------------------------------
// RGB scale of a decode, channel-pipelined (host-side runtime piece: one call instead of ~400 Python-level
// launches / event operations per decode).  Channel c's means depend on the decoded channels < c of the same
// pixel (logistic_mixture.py:262-272), so the reference codes R, G, B strictly one after the other; here the
// three serial decoders run concurrently, staggered by one chunk of pixels: chunk j of channel c-1 decoded ->
// rows of chunk j of channel c built (bld_streams[c]) -> channel c's warps resume from their saved state
// (dec_streams[c]).  Everything is ordered after what `cur_stream` has queued, and `cur_stream` waits for it.
// ---------------------------------------------------------------------------------------------
namespace {
struct EventRing {
    std::vector<cudaEvent_t> ev;
    size_t next = 0;
    cudaEvent_t get() {
        if (ev.size() < 64) {
            cudaEvent_t e = nullptr;
            if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
            ev.push_back(e);
            return e;
        }
        return ev[next++ % ev.size()];      // a wait captures the record that precedes it in host order
    }
};
}  // namespace

extern "C" int l3c_decode_rgb_pipelined(const float *l_dev, uint8_t *sym_dev, const float *targets_dev, int N, int HW,
                                        int K, int L, uint16_t *table_dev, int pitch,
                                        const l3c_dec_stream_t *const *desc_dev_per_channel, int chunk_px,
                                        void *cur_stream, void *const *bld_streams, void *const *dec_streams,
                                        int coarse) {
    L3C_REQUIRE(l_dev && sym_dev && targets_dev && table_dev && desc_dev_per_channel && bld_streams && dec_streams,
                "l3c_decode_rgb_pipelined: null pointer");
    L3C_REQUIRE(N >= 1 && HW >= 1 && chunk_px >= 1 && L == 256, "l3c_decode_rgb_pipelined: N=%d HW=%d chunk=%d L=%d", N, HW,
                chunk_px, L);
    L3C_REQUIRE(!coarse || pitch == l3c::COARSE_REC_U16, "l3c_decode_rgb_pipelined: coarse records need pitch %d, got %d",
                l3c::COARSE_REC_U16, pitch);
    thread_local EventRing rings[64];     // per host thread and device, for the lifetime of the process
    int dev_id = 0;
    L3C_CUDA(cudaGetDevice(&dev_id));
    EventRing &ring = rings[dev_id & 63];
    const int C = 3;
    cudaStream_t cur = (cudaStream_t)cur_stream;
    cudaEvent_t start = ring.get();
    L3C_REQUIRE(start != nullptr, "l3c_decode_rgb_pipelined: cudaEventCreate failed");
    L3C_CUDA(cudaEventRecord(start, cur));
    for (int c = 0; c < C; ++c) {
        L3C_CUDA(cudaStreamWaitEvent((cudaStream_t)bld_streams[c], start, 0));
        L3C_CUDA(cudaStreamWaitEvent((cudaStream_t)dec_streams[c], start, 0));
    }
    cudaEvent_t dec_done[3] = {nullptr, nullptr, nullptr};
    for (int p0 = 0; p0 < HW; p0 += chunk_px) {
        const int npx = (HW - p0 < chunk_px) ? HW - p0 : chunk_px;
        for (int c = 0; c < C; ++c) {
            cudaStream_t sb = (cudaStream_t)bld_streams[c], sd = (cudaStream_t)dec_streams[c];
            if (c > 0) L3C_CUDA(cudaStreamWaitEvent(sb, dec_done[c - 1], 0));      // this chunk of channel c-1 is decoded
            if (int e = coarse ? l3c_dmll_build_coarse(l_dev, sym_dev, targets_dev, N, HW, K, L, c, p0, npx, table_dev, sb)
                               : l3c_dmll_build_table(l_dev, sym_dev, targets_dev, N, HW, C, K, L, 1, c, p0, npx, table_dev,
                                                      pitch, sb))
                return e;
            cudaEvent_t built = ring.get();
            L3C_REQUIRE(built != nullptr, "l3c_decode_rgb_pipelined: cudaEventCreate failed");
            L3C_CUDA(cudaEventRecord(built, sb));
            L3C_CUDA(cudaStreamWaitEvent(sd, built, 0));
            if (int e = coarse ? l3c_ac_decode_streams_coarse(desc_dev_per_channel[c], N, targets_dev, (uint32_t)p0,
                                                              (uint32_t)npx, sd)
                               : l3c_ac_decode_streams(desc_dev_per_channel[c], N, L, (uint32_t)p0, (uint32_t)npx, sd))
                return e;
            dec_done[c] = ring.get();
            L3C_REQUIRE(dec_done[c] != nullptr, "l3c_decode_rgb_pipelined: cudaEventCreate failed");
            L3C_CUDA(cudaEventRecord(dec_done[c], sd));
        }
    }
    for (int c = 0; c < C; ++c) {
        L3C_CUDA(cudaStreamWaitEvent(cur, dec_done[c], 0));
        cudaEvent_t e = ring.get();
        L3C_REQUIRE(e != nullptr, "l3c_decode_rgb_pipelined: cudaEventCreate failed");
        L3C_CUDA(cudaEventRecord(e, (cudaStream_t)bld_streams[c]));
        L3C_CUDA(cudaStreamWaitEvent(cur, e, 0));
    }
    return L3C_OK;
}
