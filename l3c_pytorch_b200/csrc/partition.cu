// partition.cu -- spatial partition of the GPU (driver "green contexts", CUDA >= 12.4).
//
// The pipelined RGB decode runs two very different kinds of work at the same time: a few dozen
// latency-bound range-decoder warps (one or two per SM, each issuing a dependent instruction every few
// cycles) and the throughput-bound CDF-row builders that feed them.  When both share an SM the
// builders' warps take issue slots from the decoder warp and the serial rate of the coder drops by
// ~1.5x.  l3c_partition_streams() hands out streams that are confined to two disjoint groups of SMs,
// so the decoders own theirs.  Everything stays in the primary context (same memory, same events).
#include <cuda.h>

#include <atomic>
#include <map>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

#include "common.cuh"

namespace l3c {
namespace {

struct Driver {
    CUresult (*DeviceGet)(CUdevice *, int) = nullptr;
    CUresult (*DeviceGetDevResource)(CUdevice, CUdevResource *, CUdevResourceType) = nullptr;
    CUresult (*DevSmResourceSplitByCount)(CUdevResource *, unsigned int *, const CUdevResource *, CUdevResource *,
                                          unsigned int, unsigned int) = nullptr;
    CUresult (*DevResourceGenerateDesc)(CUdevResourceDesc *, CUdevResource *, unsigned int) = nullptr;
    CUresult (*GreenCtxCreate)(CUgreenCtx *, CUdevResourceDesc, CUdevice, unsigned int) = nullptr;
    CUresult (*GreenCtxStreamCreate)(CUstream *, CUgreenCtx, unsigned int, int) = nullptr;
    bool ok = false;
};

template <class F>
bool resolve(const char *name, F &fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
        return false;
    fn = reinterpret_cast<F>(p);
    return true;
}

const Driver &driver() {
    static Driver d = [] {
        Driver x;
        x.ok = resolve("cuDeviceGet", x.DeviceGet) && resolve("cuDeviceGetDevResource", x.DeviceGetDevResource) &&
               resolve("cuDevSmResourceSplitByCount", x.DevSmResourceSplitByCount) &&
               resolve("cuDevResourceGenerateDesc", x.DevResourceGenerateDesc) &&
               resolve("cuGreenCtxCreate", x.GreenCtxCreate) &&
               resolve("cuGreenCtxStreamCreate", x.GreenCtxStreamCreate);
        return x;
    }();
    return d;
}

struct Partition {
    int device = -1, sm_request = 0;
    int sm_a = 0, sm_b = 0;
    CUgreenCtx ctx_a = nullptr, ctx_b = nullptr;
    std::vector<CUstream> streams_a, streams_b, streams_b_low;
};

std::mutex g_mu;
std::vector<Partition *> g_parts;     // live for the life of the process

__global__ void partition_probe_kernel(int *out) {
    if (threadIdx.x == 0 && blockIdx.x == 0 && out) *out = 1;
}

}  // namespace

namespace {
// l3c_set_conv_launch_limits: 0 = no limit
std::atomic<int> g_max_sms{0}, g_conv_smem_kb{0};

int group_sm_count(cudaStream_t st) {
    std::lock_guard<std::mutex> lock(g_mu);
    for (const Partition *p : g_parts) {
        for (CUstream s : p->streams_a)
            if ((cudaStream_t)s == st) return p->sm_a;
        for (CUstream s : p->streams_b)
            if ((cudaStream_t)s == st) return p->sm_b;
        for (CUstream s : p->streams_b_low)
            if ((cudaStream_t)s == st) return p->sm_b;
    }
    return sm_count();
}

}  // namespace

// SMs a kernel launched into `st` can use: the group size for a partition stream handed out by
// l3c_partition_streams, the whole device otherwise, capped by l3c_set_conv_launch_limits (persistent kernels
// size their grid with it)
int stream_sm_count(cudaStream_t st) {
    const int n = group_sm_count(st);
    const int cap = g_max_sms.load(std::memory_order_relaxed);
    return (cap > 0 && cap < n) ? cap : n;
}

int conv_smem_kb_override() { return g_conv_smem_kb.load(std::memory_order_relaxed); }

namespace {
std::atomic<int> g_tile_schedule{0};

// Tile counters of the persistent tensor-core kernels: a slot of TILE_COUNTERS per (device, stream), so that two
// launches that can run at the same time never share one.  Launches on one stream run one after the other, and
// each launch's last claim leaves its counters at zero for the next.  Slots come from chunks of device memory
// zeroed once when the chunk is made; word 0 of a device's first chunk is its idle-CTA count.
constexpr int SLOTS_PER_CHUNK = 256;
struct CounterPool {
    std::vector<unsigned *> chunks;
    int used = 1;                                   // slot 0 of chunk 0: the idle-CTA count
    std::map<std::pair<cudaStream_t, std::thread::id>, unsigned *> slot_of;
};
CounterPool g_pools[64];
std::mutex g_pool_mu;
}  // namespace

int conv_tile_schedule() { return g_tile_schedule.load(std::memory_order_relaxed); }

int tile_counters(cudaStream_t st, int n, unsigned **counters, unsigned long long **idle_ctas) {
    L3C_REQUIRE(n >= 1 && n <= TILE_COUNTERS, "persistent tensor-core conv: %d Cout tiles (at most %d are built)", n,
                TILE_COUNTERS);
    const int dev = current_device_slot();
    std::lock_guard<std::mutex> lock(g_pool_mu);
    CounterPool &pool = g_pools[dev];
    // the per-thread default stream is one stream per host thread under one handle
    const auto key = std::make_pair(st, st == cudaStreamPerThread ? std::this_thread::get_id() : std::thread::id());
    auto it = pool.slot_of.find(key);
    if (it == pool.slot_of.end()) {
        if (pool.chunks.empty() || pool.used == SLOTS_PER_CHUNK) {
            const size_t bytes = (size_t)SLOTS_PER_CHUNK * TILE_COUNTERS * sizeof(unsigned);
            unsigned *chunk = nullptr;
            L3C_CUDA(cudaMalloc(&chunk, bytes));
            // zeroed before any kernel can use it: a one-time synchronous set
            L3C_CUDA(cudaMemset(chunk, 0, bytes));
            L3C_CUDA(cudaStreamSynchronize(0));
            pool.used = pool.chunks.empty() ? 1 : 0;
            pool.chunks.push_back(chunk);
        }
        it = pool.slot_of.emplace(key, pool.chunks.back() + (size_t)pool.used++ * TILE_COUNTERS).first;
    }
    *counters = it->second;
    *idle_ctas = reinterpret_cast<unsigned long long *>(pool.chunks[0]);
    return L3C_OK;
}

}  // namespace l3c

extern "C" int l3c_set_conv_tile_schedule(int mode) {
    L3C_REQUIRE(mode >= 0 && mode <= 2, "l3c_set_conv_tile_schedule: mode %d (0: dynamic, 1: static, 2: skewed)", mode);
    l3c::g_tile_schedule.store(mode);
    return L3C_OK;
}

extern "C" int l3c_conv_idle_ctas(long long *count, int reset) {
    using namespace l3c;
    L3C_REQUIRE(count, "l3c_conv_idle_ctas: null pointer");
    unsigned *counters = nullptr;
    unsigned long long *idle = nullptr;
    if (int e = tile_counters(0, 1, &counters, &idle)) return e;
    L3C_CUDA(cudaDeviceSynchronize());
    unsigned long long v = 0;
    L3C_CUDA(cudaMemcpy(&v, idle, sizeof(v), cudaMemcpyDeviceToHost));
    if (reset) L3C_CUDA(cudaMemset(idle, 0, sizeof(v)));
    if (reset) L3C_CUDA(cudaDeviceSynchronize());
    *count = (long long)v;
    return L3C_OK;
}

extern "C" int l3c_set_conv_launch_limits(int max_sms, int conv_smem_kb) {
    L3C_REQUIRE(max_sms >= 0 && conv_smem_kb >= 0, "l3c_set_conv_launch_limits: bad arguments (%d, %d)", max_sms,
                conv_smem_kb);
    l3c::g_max_sms.store(max_sms);
    l3c::g_conv_smem_kb.store(conv_smem_kb);
    return L3C_OK;
}

extern "C" int l3c_partition_streams2(int sm_a, int n_a, void **streams_a, int n_b_high, void **streams_b_high,
                                      int n_b_low, void **streams_b_low, int *sm_a_out, int *sm_b_out);

extern "C" int l3c_partition_streams(int sm_a, int n_a, void **streams_a, int n_b, void **streams_b,
                                     int *sm_a_out, int *sm_b_out) {
    // all but the last stream of group B are high priority, the last one has default priority
    return l3c_partition_streams2(sm_a, n_a, streams_a, n_b > 0 ? n_b - 1 : 0, streams_b, n_b > 0 ? 1 : 0,
                                  n_b > 0 ? streams_b + (n_b - 1) : nullptr, sm_a_out, sm_b_out);
}

extern "C" int l3c_partition_streams2(int sm_a, int n_a, void **streams_a, int n_b, void **streams_b,
                                      int n_b_low, void **streams_b_low, int *sm_a_out, int *sm_b_out) {
    using namespace l3c;
    L3C_REQUIRE(n_b_low >= 0 && n_b_low <= 64 && (n_b_low == 0 || streams_b_low), "l3c_partition_streams2: bad arguments");

    L3C_REQUIRE(sm_a > 0 && n_a >= 0 && n_b >= 0 && n_a <= 64 && n_b <= 64 && (n_a == 0 || streams_a) &&
                    (n_b == 0 || streams_b),
                "l3c_partition_streams: bad arguments");
    const Driver &drv = driver();
    if (!drv.ok) {
        set_error("l3c_partition_streams: this driver has no green-context API");
        return L3C_EUNSUPPORTED;
    }
    int dev = 0;
    L3C_CUDA(cudaGetDevice(&dev));
    L3C_CUDA(cudaFree(nullptr));                               // make sure the primary context exists
    std::lock_guard<std::mutex> lock(g_mu);
    Partition *part = nullptr;
    for (Partition *p : g_parts)
        if (p->device == dev && p->sm_request == sm_a) part = p;
    if (!part) {
        CUdevice cudev;
        CUdevResource all, group, rest;
        unsigned int n_groups = 1;
        CUdevResourceDesc desc_a = nullptr, desc_b = nullptr;
        Partition *p = new Partition;
        p->device = dev;
        p->sm_request = sm_a;
        const bool ok = drv.DeviceGet(&cudev, dev) == CUDA_SUCCESS &&
                        drv.DeviceGetDevResource(cudev, &all, CU_DEV_RESOURCE_TYPE_SM) == CUDA_SUCCESS &&
                        (unsigned)sm_a < all.sm.smCount &&
                        drv.DevSmResourceSplitByCount(&group, &n_groups, &all, &rest, 0, (unsigned)sm_a) == CUDA_SUCCESS &&
                        n_groups == 1 && rest.sm.smCount > 0 &&
                        drv.DevResourceGenerateDesc(&desc_a, &group, 1) == CUDA_SUCCESS &&
                        drv.DevResourceGenerateDesc(&desc_b, &rest, 1) == CUDA_SUCCESS &&
                        drv.GreenCtxCreate(&p->ctx_a, desc_a, cudev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS &&
                        drv.GreenCtxCreate(&p->ctx_b, desc_b, cudev, CU_GREEN_CTX_DEFAULT_STREAM) == CUDA_SUCCESS;
        if (!ok) {
            delete p;
            set_error("l3c_partition_streams: the driver refused to split %d SMs off device %d", sm_a, dev);
            return L3C_EUNSUPPORTED;
        }
        p->sm_a = (int)group.sm.smCount;
        p->sm_b = (int)rest.sm.smCount;
        g_parts.push_back(p);
        part = p;
    }
    // group B: all streams but the LAST one are high priority (CDF-row builders and decoder networks of the
    // decodes in flight); the last one has default priority (work that merely runs beside the decodes: the
    // encode of the next batch)
    auto grow = [&](std::vector<CUstream> &v, CUgreenCtx ctx, int n, int priority) -> bool {
        while ((int)v.size() < n) {
            CUstream s = nullptr;
            if (drv.GreenCtxStreamCreate(&s, ctx, CU_STREAM_NON_BLOCKING, priority) != CUDA_SUCCESS) return false;
            // the runtime must accept the stream: one empty launch, checked
            partition_probe_kernel<<<1, 32, 0, (cudaStream_t)s>>>(nullptr);
            if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize((cudaStream_t)s) != cudaSuccess) return false;
            v.push_back(s);
        }
        return true;
    };
    if (!grow(part->streams_a, part->ctx_a, n_a, -1) || !grow(part->streams_b, part->ctx_b, n_b, -1) ||
        !grow(part->streams_b_low, part->ctx_b, n_b_low, 0)) {
        set_error("l3c_partition_streams: could not create / use a partition stream on device %d", dev);
        return L3C_EUNSUPPORTED;
    }
    for (int i = 0; i < n_a; ++i) streams_a[i] = (void *)part->streams_a[i];
    for (int i = 0; i < n_b; ++i) streams_b[i] = (void *)part->streams_b[i];
    for (int i = 0; i < n_b_low; ++i) streams_b_low[i] = (void *)part->streams_b_low[i];
    if (sm_a_out) *sm_a_out = part->sm_a;
    if (sm_b_out) *sm_b_out = part->sm_b;
    return L3C_OK;
}
