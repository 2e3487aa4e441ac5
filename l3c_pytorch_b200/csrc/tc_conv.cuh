// tc_conv.cuh -- what the persistent tensor-core convolution kernels (conv_f16.cu, conv_tf32.cu, conv_f16x2.cu)
// share: the shared-memory stage ring of a pipe with its mbarrier protocol, the tile walk, the epilogue of the
// FP16-image 3x3 / 5x5 kernels, and the host side of a launch (tensor maps, shared-memory opt-in, stage and pipe
// planning, grid size).
//
// CTA layout: warps 0..7 are two consumer warpgroups ("pipes"), each with its own TMA producer warp (warps 8, 9),
// its own ring of shared-memory stages and its own tiles (claimed from the launch's tile queue).  A consumer
// issues wgmma on the staged operands, keeps the fp32 accumulators in registers and runs the fused epilogue
// itself, so the epilogue of one pipe overlaps the MMAs of the other.  Accumulator fragment of wgmma m64nNk*:
// thread t of the warpgroup, warp w = t / 32, lane l holds
//   d[4j + 0], d[4j + 1] = (row 16w + l/4    , columns 8j + 2*(l%4) + {0,1})
//   d[4j + 2], d[4j + 3] = (row 16w + l/4 + 8, same columns)
// Dynamic shared memory, from a 1024 B (swizzle atom) aligned start: [resident weights][pipe 0 stages]
// [pipe 1 stages][buffers of the kernel's own][barriers].
//
// Tile walk: the producer of each pipe claims tiles from a per-launch counter (one per Cout tile, blockIdx.y) with
// atomicAdd, one claim ahead, and hands each index to its consumer through a two-slot tile ring in shared memory
// before it issues the tile's TMA; so a CTA that starts late, on an SM another kernel still holds, simply runs fewer
// tiles.  Which CTA runs a tile does not change any output bit: each output's accumulation order is fixed per tile.
#pragma once
#include <initializer_list>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace l3c {
namespace tcx {

constexpr int MAX_STAGES = 4;                  // per pipe
constexpr int SMEM_MAX = 227 * 1024;           // dynamic shared memory one CTA can opt in to
constexpr int SMEM_RESERVE = 1024 + 512;       // alignment slack + barriers, part of every launch's fixed bytes
constexpr int TH = 8, TW = 16;                 // output tile of the 3x3 / 5x5 kernels: 128 pixels

// ----------------------------------------------------------------------------------------------------------------
// device side
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t *smem_aligned() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
}

// barriers at `bars` (SMEM_RESERVE keeps 512 B for them): full[MAX_STAGES], empty[MAX_STAGES] of pipe 0, the same
// of pipe 1, then the weight barrier; from +256 the tile ring of pipe k (tile_ring()): full[TQ_SLOTS],
// empty[TQ_SLOTS] at +256 + 32k, its index slots at +320 + 8k; at +336 the count of idle pipes (schedule mode 2).
constexpr int TQ_SLOTS = 2;
__device__ __forceinline__ uint32_t weight_bar(uint32_t bars) { return bars + 8u * (4 * MAX_STAGES); }
__device__ __forceinline__ uint32_t tile_ring(uint32_t bars, int k) { return bars + 256u + 32u * k; }
__device__ __forceinline__ uint32_t tile_slots(uint32_t bars, int k) { return bars + 320u + 8u * k; }
__device__ __forceinline__ uint32_t idle_pipes(uint32_t bars) { return bars + 336u; }

__device__ __forceinline__ uint64_t globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Thread 0 initialises the barriers (full: the producer's expect_tx or tile index; empty: one arrival per consumer
// warp) and prefetches both tensor maps; then the whole CTA syncs.
__device__ __forceinline__ void pipeline_init(uint32_t bars, const CUtensorMap *map_x, const CUtensorMap *map_w) {
    if (threadIdx.x == 0) {
        for (int k = 0; k < 2; ++k) {
            for (int s = 0; s < MAX_STAGES; ++s) {
                mbar_init(bars + 8u * (2 * MAX_STAGES * k + s), 1);
                mbar_init(bars + 8u * (2 * MAX_STAGES * k + MAX_STAGES + s), 4);
            }
            for (int s = 0; s < TQ_SLOTS; ++s) {
                mbar_init(tile_ring(bars, k) + 8u * s, 1);
                mbar_init(tile_ring(bars, k) + 8u * (TQ_SLOTS + s), 4);
            }
        }
        mbar_init(weight_bar(bars), 1);
        asm volatile("st.shared.u32 [%0], 0;" ::"r"(idle_pipes(bars)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(map_x) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(map_w) : "memory");
    }
    __syncthreads();
}

struct Slot {
    uint32_t dst, bar;     // stage address, its full barrier
};

// The ring of pipe k: n_stages stages of `stride` bytes from `base` (pipe 0's stages, then pipe 1's).  Producer
// and consumer each walk it with their own copy; phase flips every time the ring wraps.
struct Ring {
    uint32_t base, stride, bars, n_stages, stage, phase;

    __device__ __forceinline__ Ring(uint32_t stages_base, uint32_t stride_, uint32_t n_stages_, uint32_t bars_, int k)
        : base(stages_base + k * n_stages_ * stride_), stride(stride_), bars(bars_ + 8u * (2 * MAX_STAGES * k)),
          n_stages(n_stages_), stage(0), phase(0) {}

    __device__ __forceinline__ void advance() {
        if (++stage == n_stages) { stage = 0; phase ^= 1u; }
    }
    // producer: wait until the consumer has released the next stage, arm its full barrier for `bytes` of TMA
    __device__ __forceinline__ Slot acquire(uint32_t bytes) {
        mbar_wait(bars + 8u * (MAX_STAGES + stage), phase ^ 1u);
        const Slot s = {base + stage * stride, bars + 8u * stage};
        mbar_expect_tx(s.bar, bytes);
        advance();
        return s;
    }
    // consumer: wait until the next stage has landed; returns its address
    __device__ __forceinline__ uint32_t wait() {
        mbar_wait(bars + 8u * stage, phase);
        return base + stage * stride;
    }
    // consumer, after wgmma_wait0() and the accumulator fences: hand the stage back (one arrival per warp)
    __device__ __forceinline__ void release() {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(bars + 8u * (MAX_STAGES + stage));
        advance();
    }
};

// How the tiles of a launch are handed out (l3c_set_conv_tile_schedule)
struct TileSchedule {
    unsigned *counters;             // one per Cout tile (blockIdx.y), zero when the launch starts (modes 0, 2)
    unsigned long long *idle_ctas;  // mode 2: CTAs that ran no tile are counted here
    int mode;                       // 0: dynamic, 1: static stripe, 2: dynamic, odd CTAs start SKEW_NS late
#ifdef L3C_CTA_TRACE
    CtaTraceArg trace;              // where this launch's CTAs record themselves
#endif
};
constexpr uint64_t SKEW_NS = 500000;

#ifdef L3C_CTA_TRACE
// Diagnosis builds only (build.py --cta-trace): every CTA writes one l3c_cta_record_t (tools/cta_timeline.py).
// Thread 0 writes the start at the first instruction, pipeline_init's sync orders it before the consumers add
// their tile counts, and the latest warp to leave sets t_end.
__device__ __forceinline__ l3c_cta_record_t *trace_record(const TileSchedule &s) {
    return s.trace.rec ? s.trace.rec + blockIdx.y * gridDim.x + blockIdx.x : nullptr;
}
struct CtaTrace {
    l3c_cta_record_t *r;
    __device__ explicit CtaTrace(const TileSchedule &s) : r(trace_record(s)) {
        if (threadIdx.x != 0 || !r) return;
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        r->t_start = globaltimer();
        r->t_end = 0;
        r->smid = smid;
        r->tiles = 0;
        r->launch = (uint32_t)s.trace.launch;
        r->cta = blockIdx.y * gridDim.x + blockIdx.x;
    }
    __device__ ~CtaTrace() {
        if (r && (threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned long long *>(&r->t_end), globaltimer());
    }
};
#define L3C_TRACE_BEGIN const ::l3c::tcx::CtaTrace cta_trace_(ts)
#else
#define L3C_TRACE_BEGIN
#endif

// The tile walk of pipe k (n_pipes pipes per CTA, n_tiles tiles per Cout tile).  Producer and consumer each keep
// their own copy, as with Ring.
//   producer: first(), then claim() right after a tile's TMA is issued, so the atomic's latency overlaps the
//             stage wait; publish() hands each claimed index, and at the end -1, to the consumer before the tile's
//             TMA, so the consumer can prefetch the tile's residual while its stage is in flight.
//   consumer: take() returns the next index or -1.
// The claims of a launch on one counter number n_tiles + (its pipes): every pipe ends with exactly one failed
// claim, and the last claim of all resets the counter for the next launch on the stream.
struct TileQueue {
    uint32_t ring, slots, idle, pos, phase;
    int n_tiles, n_claimers, n_pipes, next, taken;
    TileSchedule s;

    __device__ __forceinline__ TileQueue(uint32_t bars, int k, int n_pipes_, int n_tiles_, const TileSchedule &s_)
        : ring(tile_ring(bars, k)), slots(tile_slots(bars, k)), idle(idle_pipes(bars)), pos(0), phase(0),
          n_tiles(n_tiles_), n_claimers(n_pipes_ * (int)gridDim.x), n_pipes(n_pipes_),
          next(blockIdx.x + k * gridDim.x), taken(0), s(s_) {}

    __device__ __forceinline__ void advance() {
        if (++pos == TQ_SLOTS) { pos = 0; phase ^= 1u; }
    }
    __device__ __forceinline__ int claim() {
        if (s.mode == 1) {                       // static stripe: pipes of a CTA take alternate tiles of its sequence
            const int t = next;
            next += n_claimers;
            return t < n_tiles ? t : -1;
        }
        unsigned *c = s.counters + blockIdx.y;
        const unsigned v = atomicAdd(c, 1u);
        if (v == (unsigned)(n_tiles + n_claimers - 1)) atomicExch(c, 0u);
        return v < (unsigned)n_tiles ? (int)v : -1;
    }
    __device__ __forceinline__ int first() {
        if (s.mode == 2 && (blockIdx.x & 1)) {
            const uint64_t t0 = globaltimer();
            while (globaltimer() - t0 < SKEW_NS) __nanosleep(1000);
        }
        return claim();
    }
    __device__ __forceinline__ void publish(int t) {
        mbar_wait(ring + 8u * (TQ_SLOTS + pos), phase ^ 1u);
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(slots + 4u * pos), "r"(t) : "memory");
        mbar_arrive(ring + 8u * pos);
        advance();
    }
    __device__ __forceinline__ int take() {
        mbar_wait(ring + 8u * pos, phase);
        int t;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(t) : "r"(slots + 4u * pos) : "memory");
        __syncwarp();
        if ((threadIdx.x & 31) == 0) mbar_arrive(ring + 8u * (TQ_SLOTS + pos));
        advance();
        const bool leader = (threadIdx.x & 127) == 0;
        if (t >= 0) {
            ++taken;
            return t;
        }
#ifdef L3C_CTA_TRACE
        if (leader && trace_record(s)) atomicAdd(&trace_record(s)->tiles, (unsigned)taken);
#endif
        if (s.mode == 2 && taken == 0 && leader) {
            // idle pipes count themselves; the CTA is idle when all n_pipes of them did
            uint32_t before;
            asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(before) : "r"(idle) : "memory");
            if ((int)before == n_pipes - 1) atomicAdd(s.idle_ctas, 1ull);
        }
        return t;
    }
};

// producer: claim tiles, publish each and then the end, call f(t) to issue tile t's TMA
template <class F>
__device__ __forceinline__ void produce_tiles(TileQueue &q, F &&f) {
    for (int t = q.first();; t = q.claim()) {
        q.publish(t);
        if (t < 0) return;
        f(t);
    }
}
// consumer: f(t) for every tile the producer publishes
template <class F>
__device__ __forceinline__ void consume_tiles(TileQueue &q, F &&f) {
    for (int t = q.take(); t >= 0; t = q.take()) f(t);
}

// 3x3 / 5x5 layers (conv3x3_tf32_kernel, conv_f16_kernel, conv3x3_f16x2_kernel)
struct Params {
    const float *bias;      // padded to cout_pad
    const float *residual;  // fp32, layout of y, or null
    float *y;               // fp32 output or null
    float *y_tf32;          // tf32: TF32-rounded twin of y or null
    __half *yh;             // f16: FP16 image of the output, f16x2: split image; or null
    int N, H, W;            // H, W: the output pixels the tiles cover
    int Cout, y_pitch, y_coff;
    int yh_pitch, yh_lo_off;   // f16x2: pitch of the split image, offset of its lo plane
    int dilation;
    unsigned flags;
    int tiles_x, tiles_y;
};

struct Tile {
    int tx, ty, n;
};
__device__ __forceinline__ Tile tile_of(const Params &p, int t) {
    return {t % p.tiles_x, t / p.tiles_x % p.tiles_y, t / p.tiles_x / p.tiles_y};
}

// Which pixels of an 8x16 tile the two 64-row halves (acc[0], acc[1]) of the MMA are.
//   ROWS: half h = tile rows 4h..4h+3 (8-row group g = row 4h + g/2, pixels 8(g%2)..+7): conv3x3_f16x2_kernel and
//         the 5x5/s2 kernel, whose boxes are 16 px wide
//   COLS: half h = pixels 8h..8h+7 of all 8 rows (group g = row g): the 3x3 f16 kernel, whose groups are evenly
//         spaced rows of one wide halo box
// Accumulator row 16w + tr + 8rh of half h (consumer warp w, tr = lane / 4) is tile row half_row(), pixel half_px().
enum class Halves { ROWS, COLS };
template <Halves HV>
__device__ __forceinline__ int half_row(int h, int w, int rh) { return HV == Halves::ROWS ? 4 * h + w : 2 * w + rh; }
template <Halves HV>
__device__ __forceinline__ int half_px(int h, int tr, int rh) { return HV == Halves::ROWS ? tr + 8 * rh : 8 * h + tr; }

// fp32 pair -> operand image: FP16 pair, or with SPLIT its hi and lo pairs
template <bool SPLIT>
__device__ __forceinline__ void to_image(float a, float b, uint32_t &hi, uint32_t &lo) {
    if (SPLIT) split_h2(a, b, hi, lo);
    else hi = pack_h2(a, b);
}

// L2 prefetch of the fp32 residual lines image_epilogue() reads for tile c of Cout tile ct, consumer warp w
// (one 128 B line per pixel and column half, issued by the first lane of each quad).  Issued before the tile's
// MMAs, so that the epilogue's residual loads find their lines in L2 instead of waiting on HBM.  Without
// residual or with PixelShuffle(2) (no residual there) nothing is fetched.
template <Halves HV>
__device__ __forceinline__ void prefetch_residual(const Params &p, const Tile &c, int ct, int w) {
    if (p.residual == nullptr || (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0 || (threadIdx.x & 3) != 0) return;
    const int tr = (threadIdx.x & 31) >> 2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
            const int oy = c.ty * TH + half_row<HV>(h, w, rh);
            const int ox = c.tx * TW + half_px<HV>(h, tr, rh);
            if (oy >= p.H || ox >= p.W) continue;
            const size_t pix = ((size_t)c.n * p.H + oy) * p.W + ox;
#pragma unroll
            for (int cc = 0; cc < 2; ++cc)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + pix * p.y_pitch + p.y_coff + ct * 64 + 32 * cc));
        }
    }
}

// Epilogue of the FP16-image 3x3 / 5x5 kernels (conv_f16_kernel, conv3x3_f16x2_kernel; SPLIT: f16x2) for tile c of
// Cout tile ct, consumer warp w; acc[h] holds the conv values of tile half h (HV: which pixels that is).  Adds the
// bias, ReLU, the fp32 residual, and writes the fp32 output (float2: full sectors) and the operand image (16-byte
// vectors after a 4x4 transpose inside each quad; SPLIT: hi and lo planes yh_lo_off apart), or PixelShuffle(2) of
// both.  Fragment (h, column half cc, rh) = tile row half_row(h, w, rh), pixel half_px(h, tr, rh), columns
// 32cc + 8jb + 2tq; either way the eight lanes tr of a fragment hold eight consecutive pixels of one row.
template <bool SPLIT, Halves HV>
__device__ __forceinline__ void image_epilogue(const Params &p, const Tile &c, int ct, int w, const float (&acc)[2][32]) {
    const int lane = threadIdx.x & 31, tq = lane & 3, tr = lane >> 2;   // column pair / row inside the fragment
    const bool relu = (p.flags & L3C_CONV_RELU) != 0;
    const bool shuffle = (p.flags & L3C_CONV_PIXEL_SHUFFLE2) != 0;
    const int hp = SPLIT ? p.yh_pitch : p.y_pitch;                        // pitch of the operand image
    // Without SPLIT the residual of a tile half is loaded before the half's first store: the compiler cannot tell
    // that y / yh do not alias it, so a load left inside the loop waits behind every store before it (one L2 round
    // trip per fragment instead of one per half).  The whole tile's residual at once would exceed the 168
    // registers a thread has; in the split kernel, whose registers are already short, even a half's spills.
    const bool add_res = p.residual != nullptr && !shuffle;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float2 res[2][2][4];                                              // [cc][rh][jb]
        if (!SPLIT && add_res) {
#pragma unroll
            for (int cc = 0; cc < 2; ++cc)
#pragma unroll
                for (int rh = 0; rh < 2; ++rh) {
                    const int oy = c.ty * TH + half_row<HV>(h, w, rh);
                    const int ox = c.tx * TW + half_px<HV>(h, tr, rh);
                    const size_t off = (((size_t)c.n * p.H + oy) * p.W + ox) * p.y_pitch + p.y_coff + ct * 64 + 32 * cc;
#pragma unroll
                    for (int jb = 0; jb < 4; ++jb)
                        res[cc][rh][jb] = (oy < p.H && ox < p.W)
                                              ? __ldg(reinterpret_cast<const float2 *>(p.residual + off + 8 * jb + 2 * tq))
                                              : make_float2(0.f, 0.f);
                }
        }
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
            const int cb = ct * 64 + 32 * cc;                             // first conv channel of this fragment
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int oy = c.ty * TH + half_row<HV>(h, w, rh);
                const int ox = c.tx * TW + half_px<HV>(h, tr, rh);
                const bool inside = (oy < p.H) && (ox < p.W);
                const size_t pix = ((size_t)c.n * p.H + oy) * p.W + ox;
                float a[4], b[4];
#pragma unroll
                for (int jb = 0; jb < 4; ++jb) {
                    const float2 bb = __ldg(reinterpret_cast<const float2 *>(p.bias + cb + 8 * jb + 2 * tq));
                    a[jb] = acc[h][16 * cc + 4 * jb + 2 * rh] + bb.x;
                    b[jb] = acc[h][16 * cc + 4 * jb + 2 * rh + 1] + bb.y;
                    if (relu) { a[jb] = fmaxf(a[jb], 0.f); b[jb] = fmaxf(b[jb], 0.f); }
                }
                if (!shuffle) {
                    const size_t off = pix * p.y_pitch + p.y_coff + cb;
                    if (add_res && inside) {
#pragma unroll
                        for (int jb = 0; jb < 4; ++jb) {
                            const float2 r = SPLIT ? __ldg(reinterpret_cast<const float2 *>(p.residual + off + 8 * jb + 2 * tq))
                                                   : res[cc][rh][jb];
                            a[jb] += r.x; b[jb] += r.y;
                        }
                    }
                    if (p.y != nullptr && inside) {
#pragma unroll
                        for (int jb = 0; jb < 4; ++jb)
                            *reinterpret_cast<float2 *>(p.y + off + 8 * jb + 2 * tq) = make_float2(a[jb], b[jb]);
                    }
                    if (p.yh != nullptr) {
                        uint32_t hv[4], lv[4];
#pragma unroll
                        for (int jb = 0; jb < 4; ++jb) to_image<SPLIT>(a[jb], b[jb], hv[jb], lv[jb]);
                        quad_transpose(hv, tq);               // -> channels cb + 8*tq + 0..7
                        if (SPLIT) quad_transpose(lv, tq);
                        if (inside) {
                            const size_t oh = pix * hp + p.y_coff + cb + 8 * tq;
                            *reinterpret_cast<uint4 *>(p.yh + oh) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
                            if (SPLIT) *reinterpret_cast<uint4 *>(p.yh + oh + p.yh_lo_off) = make_uint4(lv[0], lv[1], lv[2], lv[3]);
                        }
                    }
                } else {
                    // out[n, 2*oy+si, 2*ox+sj, cq] = conv[n, oy, ox, 4*cq + 2*si + sj]   (edsr.py:92-101)
                    const size_t W2 = 2 * (size_t)p.W;
                    const size_t row0 = ((size_t)c.n * (2 * p.H) + 2 * oy) * W2 + 2 * ox;   // output pixel (si=0, sj=0)
                    // after the transpose thread tq owns conv channels c0 + 0..7 (c0 = cb + 8*tq) = output channels
                    // cq0, cq0 + 1 of the four sub-pixels, and a quad writes 32 contiguous bytes per output pixel
                    uint32_t fa[4], fb[4];
#pragma unroll
                    for (int jb = 0; jb < 4; ++jb) { fa[jb] = __float_as_uint(a[jb]); fb[jb] = __float_as_uint(b[jb]); }
                    quad_transpose(fa, tq);                   // fa[s] = channel c0 + 2s, fb[s] = channel c0 + 2s + 1
                    quad_transpose(fb, tq);
                    if (inside) {
                        const int cq0 = (cb + 8 * tq) >> 2;
#pragma unroll
                        for (int si = 0; si < 2; ++si) {
                            const float x00 = __uint_as_float(fa[si]), x01 = __uint_as_float(fa[2 + si]);   // sj = 0: cq0, cq0+1
                            const float x10 = __uint_as_float(fb[si]), x11 = __uint_as_float(fb[2 + si]);   // sj = 1
                            if (p.y != nullptr) {
                                const size_t o2 = (row0 + si * W2) * p.y_pitch + p.y_coff + cq0;
                                *reinterpret_cast<float2 *>(p.y + o2) = make_float2(x00, x01);
                                *reinterpret_cast<float2 *>(p.y + o2 + p.y_pitch) = make_float2(x10, x11);
                            }
                            if (p.yh != nullptr) {
                                const size_t oh = (row0 + si * W2) * hp + p.y_coff + cq0;
                                uint32_t h0, l0, h1, l1;
                                to_image<SPLIT>(x00, x01, h0, l0);
                                to_image<SPLIT>(x10, x11, h1, l1);
                                *reinterpret_cast<uint32_t *>(p.yh + oh) = h0;
                                if (SPLIT) *reinterpret_cast<uint32_t *>(p.yh + oh + p.yh_lo_off) = l0;
                                *reinterpret_cast<uint32_t *>(p.yh + oh + hp) = h1;
                                if (SPLIT) *reinterpret_cast<uint32_t *>(p.yh + oh + hp + p.yh_lo_off) = l1;
                            }
                        }
                    }
                }
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------------------------

// Params of a 3x3 / 5x5 launch whose tiles cover H x W output pixels
static inline Params conv_params(const l3c_conv_t &p, int H, int W) {
    Params q;
    q.bias = p.bias; q.residual = p.residual; q.y = p.y; q.y_tf32 = p.y_tf32;
    q.yh = reinterpret_cast<__half *>(p.y_h);
    q.N = p.N; q.H = H; q.W = W;
    q.Cout = p.Cout; q.y_pitch = p.y_pitch; q.y_coff = p.y_coff;
    q.yh_pitch = p.yh_pitch; q.yh_lo_off = p.yh_lo_off;
    q.dilation = p.dilation; q.flags = p.flags;
    q.tiles_x = ceil_div(W, TW);
    q.tiles_y = ceil_div(H, TH);
    return q;
}

// TMA map of a dense tensor at `base` as the kernels read it: 128B swizzle, 128 B L2 promotion, zero fill out of
// bounds (the conv padding).  dims innermost first, strides in bytes of dims 1.., box in elements, element strides
// 1 unless given.  On failure sets the error (`who`: the entry point, `what`: the operand) and returns false.
inline bool encode_tmap(CUtensorMap *map, const char *who, const char *what, CUtensorMapDataType dt, const void *base,
                        std::initializer_list<long long> dims, std::initializer_list<long long> strides,
                        std::initializer_list<int> box, std::initializer_list<int> estr = {}) {
    typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                      const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiledFn encode = nullptr;
    if (!encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            encode = reinterpret_cast<EncodeTiledFn>(fn);
    }
    if (!encode) {
        set_error("%s: cuTensorMapEncodeTiled is not available from the driver", who);
        return false;
    }
    const int rank = (int)dims.size();
    cuuint64_t d[5], s[5];
    cuuint32_t b[5], e[5];
    for (int i = 0; i < rank; ++i) {
        d[i] = (cuuint64_t)dims.begin()[i];
        s[i] = i + 1 < rank ? (cuuint64_t)strides.begin()[i] : 0;
        b[i] = (cuuint32_t)box.begin()[i];
        e[i] = estr.size() ? (cuuint32_t)estr.begin()[i] : 1;
    }
    const CUresult r = encode(map, dt, rank, const_cast<void *>(base), d, s, b, e, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("%s: cuTensorMapEncodeTiled(%s) failed with %d", who, what, (int)r);
        return false;
    }
    return true;
}

struct RingPlan {
    int n_pipes, n_stages, smem_bytes;   // n_stages == 0: the layer does not fit
};

// Stages per pipe: as many as fit in `budget` beside `fixed` bytes (resident weights, the kernel's own buffers,
// SMEM_RESERVE) with two pipes, at most max_stages.  If not even one fits: one stage per pipe above the budget if
// two pipes fit in SMEM_MAX, else one pipe with one stage where the kernel can run with one pipe.
static inline RingPlan plan_ring(int budget, int fixed, int stage_bytes, int max_stages, bool one_pipe_ok = false) {
    int n = (budget - fixed) / (2 * stage_bytes);
    if (n > max_stages) n = max_stages;
    if (n < 1 && fixed + 2 * stage_bytes <= SMEM_MAX) n = 1;
    if (n >= 1) return {2, n, fixed + 2 * n * stage_bytes};
    if (one_pipe_ok && fixed + stage_bytes <= SMEM_MAX) return {1, 1, fixed + stage_bytes};
    return {2, 0, 0};
}

// 3x3 / 5x5 grid: gridDim.y = Cout tiles (resident weights), gridDim.x = the stream's SMs shared among them, at
// least 1 and at most one CTA per pixel tile
static inline dim3 grid_3x3(cudaStream_t st, int cout_tiles, int ptiles) {
    int per_ct = stream_sm_count(st) / cout_tiles;
    if (per_ct < 1) per_ct = 1;
    if (per_ct > ptiles) per_ct = ptiles;
    return dim3(per_ct, cout_tiles);
}

// 1x1 grid: two pipes per CTA, at most one CTA per SM of the stream
static inline int grid_1x1(cudaStream_t st, int n_tiles) {
    const int n_sm = stream_sm_count(st);
    return ceil_div(n_tiles, 2) < n_sm ? ceil_div(n_tiles, 2) : n_sm;
}

// Launches a persistent tensor-core kernel under `name` (the launch log), its tile schedule (the stream's tile
// counters) as the last argument.  The opt-in to SMEM_MAX bytes of dynamic shared memory is per device, so it is
// done once per device and kernel.
template <auto Kernel, class... Args>
int launch_tc(const char *name, dim3 grid, int smem_bytes, cudaStream_t st, const Args &...args) {
    static bool configured_dev[64] = {};
    bool &configured = configured_dev[current_device_slot()];
    if (!configured) {
        L3C_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
        configured = true;
    }
    TileSchedule ts;
    ts.mode = conv_tile_schedule();
    if (int e = tile_counters(st, (int)grid.y, &ts.counters, &ts.idle_ctas)) return e;
#ifdef L3C_CTA_TRACE
    ts.trace = cta_trace_launch(name, grid, st);
#endif
    Kernel<<<grid, THREADS, smem_bytes, st>>>(args..., ts);
    L3C_LAUNCH_CHECK(name);
    return L3C_OK;
}

}  // namespace tcx
}  // namespace l3c
