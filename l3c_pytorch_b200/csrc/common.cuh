// common.cuh -- shared helpers for libl3c_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include <initializer_list>

#include "../../include/l3c_b200.h"

namespace l3c {

void set_error(const char *fmt, ...);

#define L3C_REQUIRE(cond, ...)                      \
    do {                                            \
        if (!(cond)) {                              \
            ::l3c::set_error(__VA_ARGS__);          \
            return L3C_EINVAL;                      \
        }                                           \
    } while (0)

#define L3C_CUDA(call)                                                                   \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess) {                                                        \
            ::l3c::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),    \
                             __FILE__, __LINE__);                                        \
            return L3C_ECUDA;                                                            \
        }                                                                                \
    } while (0)

#define L3C_LAUNCH_CHECK(name)                                                           \
    do {                                                                                 \
        cudaError_t e__ = cudaGetLastError();                                            \
        if (e__ != cudaSuccess) {                                                        \
            ::l3c::set_error("launch of %s failed: %s", name, cudaGetErrorString(e__));  \
            return L3C_ECUDA;                                                            \
        }                                                                                \
        ::l3c::count_launch(name);                                                       \
    } while (0)

void count_launch(const char *kernel_name);   // per-kernel launch counters (l3c_launch_log)

// 1x1 layers with Cin % 64 == 0 on the tensor cores, all three tensor-core precisions (conv_f16.cu)
int conv1x1_tc(const l3c_conv_t &p, cudaStream_t st);

// Argument checks of the 3x3 backward passes (conv_train.cu): every pointer non-null and 16-byte aligned, Cin 64,
// Cout 64 or 256, dilation 1, 2 or 4, N in [1, 65535], H * W <= 2^30.  L3C_EINVAL with the message otherwise.
int conv3x3_backward_args(const char *fn, std::initializer_list<const void *> ptrs, int N, int H, int W, int Cin,
                          int Cout, int dilation);

int sm_count();                          // SMs of the current device
int stream_sm_count(cudaStream_t st);    // SMs available to kernels launched into `st` (partition.cu)
int conv_smem_kb_override();             // l3c_set_conv_launch_limits' conv_smem_kb, 0 = none (partition.cu)
int conv_tile_schedule();                // l3c_set_conv_tile_schedule's mode (partition.cu)
// The tile counters of a persistent tensor-core launch into `st` (n <= TILE_COUNTERS of them, zero; no stream but
// `st` uses them) and the device's idle-CTA count of schedule mode 2 (partition.cu)
constexpr int TILE_COUNTERS = 32;
int tile_counters(cudaStream_t st, int n, unsigned **counters, unsigned long long **idle_ctas);

#ifdef L3C_CTA_TRACE
// diagnosis builds: where the CTAs of the next launch record themselves (rec null: not recorded) (capi.cu)
struct CtaTraceArg {
    l3c_cta_record_t *rec;
    int launch;
};
CtaTraceArg cta_trace_launch(const char *name, dim3 grid, cudaStream_t st);
#endif

// cudaFuncSetAttribute is per DEVICE: "done once" flags must be kept per device, or a process that drives a second
// GPU launches its kernels there without the opt-in for > 48 KB of dynamic shared memory
static inline int current_device_slot() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev & 63;
}

// row pitch of the decoder's tables: 32 entries for L <= 32, 256 up to L = 256, else L rounded up to a multiple of 8
__host__ __device__ static inline int decode_pitch(int L) { return (L <= 32) ? 32 : (L <= 256) ? 256 : (L + 7) & ~7; }

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// n items of `per` threads each, in CTAs of 256 threads, fit in one grid row: at most 2^31 - 1 CTAs (CUDA's
// grid.x limit; a larger count cast to the launch's unsigned would silently cover only part of the items)
static inline bool fits_grid_x(int64_t n, int64_t per = 1) { return n >= 0 && n <= 0x7fffffffll * 256 / per; }

}  // namespace l3c
