// range_coder.cu -- batched binary arithmetic coder for sm_90a: one coding warp per stream (decoders of L > 32 and the
// encoder: plus a helper / emitter warp).
//
// Bit-exact re-statement of the reference coder's integer arithmetic
//   encoder: /root/reference/src/torchac/torchac_backend/torchac.cpp:152-227 (+ bit sink :63-93)
//   decoder: /root/reference/src/torchac/torchac_backend/torchac.cpp:299-381 (+ :96-128, :276-296)
// re-designed for the GPU:
//   * the reference's bit-at-a-time renormalisation loops are collapsed into two count-leading-
//     zeros steps (all "equal MSB" shifts first, then all "underflow" shifts -- the reference loop
//     can only ever visit them in that order, see DESIGN.md section 4.4);
//   * the encoder consumes pre-computed 32-bit (c_low, c_high-1) intervals (one coalesced load per
//     32 symbols) instead of indexing a CDF table with the symbol;
//   * the encoder keeps bit emission off its serial chain and off its warp: per symbol only (low, k, u) is
//     recorded, every 32 symbols an emitter warp packs the 32 bit strings in parallel (one packed scan);
//   * the decoder replaces the per-row binary search by a warp-wide comparison of the whole CDF row
//     against the code value (no division: cdf[m] <= ((value-low+1)*2^16-1)/span  <=>
//     mulhi(cdf[m] << 16, span) <= value - low) and one warp max-reduction over packed
//     (cdf[m], cdf[m+1]-1) proposals; rows are prefetched one to two groups of 8 symbols ahead so
//     HBM latency stays off the serial dependency chain;
//   * coder state is (low, r = high - low[, dv = value - low]): every renormalisation shift maps
//     r -> 2r+1, dv -> 2dv+bit, so `high`, `value` and the MSB fix-ups leave the chain;
//   * coder state can be saved/restored so that a stream may be decoded in chunks while later CDF
//     rows are still being built (RGB channel pipelining).
#include <stdlib.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "common.cuh"
#include "dmll_math.cuh"

namespace l3c {

constexpr unsigned FULL = 0xFFFFFFFFu;

// shared-memory hand-over between the warps of a stream (the encoder's and the decoders' rings)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}

// ---------------------------------------------------------------------------------------------
// encoder
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t shl_c(uint32_t x, uint32_t n) {   // x << n, 0 for n >= 32 (PTX clamps)
    uint32_t r;
    asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(n));
    return r;
}
__device__ __forceinline__ uint32_t shr_c(uint32_t x, uint32_t n) {   // x >> n, 0 for n >= 32
    uint32_t r;
    asm("shr.u32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(n));
    return r;
}
__device__ __forceinline__ uint32_t clz_nz(uint32_t x) {             // count leading zeros, x != 0
    uint32_t r;
    asm("bfind.shiftamt.u32 %0, %1;" : "=r"(r) : "r"(x));
    return r;
}
struct BitSink {
    uint32_t *out;       // word pointer (big-endian words)
    uint32_t cap_words;
    uint32_t wpos;
    uint64_t acc;
    int nacc;            // < 32 between calls
    int lane;

    __device__ __forceinline__ void put(uint32_t v, int n) {   // 0 <= n <= 32, v < 2^n
        acc = (acc << n) | v;
        nacc += n;
        if (nacc >= 32) {
            const uint32_t w = (uint32_t)(acc >> (nacc - 32));
            if (lane == 0 && wpos < cap_words) out[wpos] = __byte_perm(w, 0, 0x0123);
            wpos++;
            nacc -= 32;
        }
    }
    __device__ __forceinline__ void put_run(uint32_t bit, uint32_t count) {
        const uint32_t ones = bit ? 0xFFFFFFFFu : 0u;
        while (count >= 32) {
            put(ones, 32);
            count -= 32;
        }
        if (count) put(ones & ((1u << count) - 1u), (int)count);
    }
};

// Emission is kept OFF the coder's serial dependency chain and off its warp: the coding warp only
// records, per symbol, the pre-shift `low` and the two shift counts (k decided bits, u underflow shifts)
// in lane j's registers and hands every 32 records to the stream's emitter warp through a shared-memory
// ring; the emitter turns the 32 records into bits IN PARALLEL:
//   pending(j)  = underflow bits owed when symbol j is reached  (segmented sum of u, reset by k > 0)
//   string(j)   = k(j) > 0 ?  b0, pending(j) x !b0, remaining k-1 bits  :  nothing   (torchac.cpp:186-206)
//   offset(j)   = exclusive prefix sum of the string lengths
// one packed warp scan gives all three, the strings are OR-ed into a shared-memory staging area and
// the completed words are stored coalesced.  Batches containing a run of more than 31 owed bits take
// the sequential sink instead (rare; same bits).
constexpr int STAGE_WORDS = 68;      // 31 carried bits + 32 strings of <= 63 bits, + 2 words of slack

struct Emitter {
    uint32_t *stage;     // shared memory, STAGE_WORDS words, private to the warp
    BitSink sink;
    uint32_t pending;    // underflow bits owed (torchac.cpp:165)

    // sequential path: exactly the reference's order of operations
    __device__ __forceinline__ void emit_serial(uint32_t rec_low, uint32_t k, uint32_t u) {
        for (int j = 0; j < 32; ++j) {
            const uint32_t kj = __shfl_sync(FULL, k, j);
            const uint32_t uj = __shfl_sync(FULL, u, j);
            const uint32_t lj = __shfl_sync(FULL, rec_low, j);
            const uint32_t top_bits = shr_c(lj, 32u - kj);
            if (pending == 0u || kj == 0u) {
                sink.put(top_bits, (int)kj);
            } else {
                const uint32_t b0 = top_bits >> (kj - 1u);
                sink.put(b0, 1);
                sink.put_run(b0 ^ 1u, pending);
                pending = 0u;
                sink.put(top_bits & ~(1u << (kj - 1u)), (int)kj - 1);
            }
            pending += uj;
        }
    }

    // one record per lane (k = u = 0 for lanes without a symbol)
    __device__ __forceinline__ void emit(uint32_t rec_low, uint32_t k, uint32_t u) {
        const int lane = sink.lane;
        const uint32_t own = k | (u << 16);
        uint32_t x = own;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(FULL, x, d);
            if (lane >= d) x += y;
        }
        const uint32_t excl = x - own;
        const uint32_t fmask = __ballot_sync(FULL, k > 0u);
        const uint32_t below = fmask & ((1u << lane) - 1u);
        const uint32_t at_last = __shfl_sync(FULL, excl, (31 - __clz((int)below)) & 31);
        const uint32_t tot = __shfl_sync(FULL, x, 31);
        const uint32_t at_lastall = __shfl_sync(FULL, excl, (31 - __clz((int)fmask)) & 31);
        // owed bits when this lane's symbol is reached / bits emitted by the lanes before it
        const uint32_t pend_before = below ? (excl >> 16) - (at_last >> 16) : pending + (excl >> 16);
        const uint32_t off = (excl & 0xFFFFu) + (below ? pending + (at_last >> 16) : 0u);
        const uint32_t total_bits = (tot & 0xFFFFu) + (fmask ? pending + (at_lastall >> 16) : 0u);
        const uint32_t new_pending = fmask ? (tot >> 16) - (at_lastall >> 16) : pending + (tot >> 16);
        if (__builtin_expect(__any_sync(FULL, k > 0u && pend_before > 31u), 0)) {
            emit_serial(rec_low, k, u);
            return;
        }
        const uint32_t nacc = (uint32_t)sink.nacc;
        stage[lane] = (lane == 0 && nacc) ? (uint32_t)(sink.acc << (32u - nacc)) : 0u;
        stage[lane + 32] = 0u;
        if (lane < STAGE_WORDS - 64) stage[lane + 64] = 0u;
        __syncwarp();
        if (k > 0u) {
            const uint32_t T = rec_low >> (32u - k);
            uint64_t str = T;
            uint32_t len = k;
            if (pend_before) {
                const uint32_t b0 = T >> (k - 1u);
                const uint32_t rest = T & ~(1u << (k - 1u));
                const uint32_t run = b0 ? 0u : ((1u << pend_before) - 1u);
                str = ((((uint64_t)b0 << pend_before) | run) << (k - 1u)) | rest;
                len = k + pend_before;                                   // <= 63
            }
            const uint64_t X = str << (64u - len);                       // left-aligned
            const uint32_t P = nacc + off;
            const uint32_t w = P >> 5, b = P & 31u;
            const uint32_t w0 = (uint32_t)(X >> 32) >> b;
            const uint32_t w1 = (uint32_t)((X << (32u - b)) >> 32);
            const uint32_t w2 = b ? (uint32_t)((X << (64u - b)) >> 32) : 0u;
            if (w0) atomicOr(stage + w, w0);
            if (w1) atomicOr(stage + w + 1, w1);
            if (w2) atomicOr(stage + w + 2, w2);
        }
        __syncwarp();
        const uint32_t end = nacc + total_bits;
        const uint32_t full = end >> 5;                                  // <= 63 completed words
        for (uint32_t i = lane; i < full; i += 32) {
            if (sink.wpos + i < sink.cap_words) sink.out[sink.wpos + i] = __byte_perm(stage[i], 0, 0x0123);
        }
        const uint32_t partial = stage[full];
        sink.wpos += full;
        sink.nacc = (int)(end & 31u);
        sink.acc = sink.nacc ? (uint64_t)(partial >> (32 - sink.nacc)) : 0ull;
        pending = new_pending;
        __syncwarp();
    }
};

constexpr int ENC_RING = 4;          // ring slots of 32 records between a stream's coding and emitter warps

// (x << n) >> 32 for a 64-bit x and n <= 32 (the clamp keeps n = 32 exact: the low word)
__device__ __forceinline__ uint32_t shl64_hi(uint64_t x, uint32_t n) {
    uint32_t r;
    asm("shf.l.clamp.b32 %0, %1, %2, %3;" : "=r"(r) : "r"((uint32_t)x), "r"((uint32_t)(x >> 32)), "r"(n));
    return r;
}

// Coding warp.  Coder state is (low, r = high - low): `high` itself is never needed.  Every renormalisation
// shift -- "equal MSB" (low <<= 1, high = high << 1 | 1) or "underflow" (the same with the MSBs forced to 0 / 1)
// -- maps r to 2r + 1 (mod 2^32) and leaves bit 31 of low clear, so
//     r' + 1 = width << s,   low' = (low << s) & 0x7FFFFFFF      with width = hi16 - lo16, s = k + u.
// The next symbol's products span' * c are therefore (width * c) << s: they are formed as soon as width is known,
// beside the clz chain that yields s, and s only shifts them (one funnel shift each).  The state carried from one
// symbol to the next is (low before its shift, s, and the two products pre-shifted by 16): the interval bounds are
// bits 16..47 of product << s, the high word of (product << 16) << s.  A stream starts at span 2^32 = 1 << 32.
// This equals the r-recurrence of torchac.cpp mod 2^32 whenever the true width << s <= 2^32, i.e. on every valid
// interval (c_lo < c_hi); a width of 2^32 (c_lo = 0, c_hi = 65536 at span 2^32) is kept as (width - 1) * c + c.
// The shifted low is not masked to 31 bits on the chain: its bit 31 only flips bit 31 of low and high, which leaves
// low ^ high (k), the underflow bits below the first differing one (u) and every later low's bits 0..30 unchanged;
// the record and the terminator clear it.
// SEEK (l3c_ac_encode_streams_seek): before symbol j = every, 2 every, ... < n (every a multiple of 32: the start of a
// batch), lane 0 writes the decoder's low and high to words 0 and 1 of point j / every - 1 at `pts`; the width of the
// previous symbol gives high: r + 1 = width << s.
template <bool SEEK = false>
__device__ __forceinline__ void encode_records(const uint32_t *__restrict__ iv, uint32_t n, uint2 (*ring)[32],
                                               uint32_t bar0, int lane, uint32_t every = 0u,
                                               uint32_t *__restrict__ pts = nullptr) {
    uint32_t next = (lane < n) ? __ldg(iv + lane) : 0u;
    uint32_t lowp = 0u, s = 32u;
    uint32_t wlast = 0u;                                   // SEEK: width - 1 of the last symbol coded
    uint64_t xl, xh;
    {
        const uint32_t v = __shfl_sync(FULL, next, 0);
        xl = (uint64_t)(v & 0xFFFFu) << 16;
        xh = (uint64_t)((v >> 16) + 1u) << 16;
    }

    // one coding step (torchac.cpp:171-206); lane j keeps the record of symbol j of the batch
#define L3C_ENC_STEP(j)                                                                                            \
    {                                                                                                              \
        const uint32_t v1 = __shfl_sync(FULL, (j) < 31 ? mine : next, ((j) + 1) & 31);   /* the next symbol */     \
        const uint32_t c_lo1 = v1 & 0xFFFFu;                                                                       \
        const uint32_t c_hi1 = (v1 >> 16) + 1u;                                                                    \
        const uint32_t lo16 = shl64_hi(xl, s);                                                                     \
        const uint32_t hi16 = shl64_hi(xh, s);                                                                     \
        const uint32_t lowm = shl_c(lowp, s);                           /* bit 31 unmasked, see above */           \
        const uint32_t low = lowm + lo16;                                                                          \
        const uint32_t high = lowm + hi16 - 1u;                                                                    \
        const uint32_t wm1 = hi16 - lo16 - 1u;                           /* width - 1 */                           \
        xl = ((uint64_t)wm1 * c_lo1 + c_lo1) << 16;                                                                \
        xh = ((uint64_t)wm1 * c_hi1 + c_hi1) << 16;                                                                \
        /* renormalisation: k "equal MSB" shifts, then u "underflow" shifts */                                     \
        const uint32_t d = low ^ high;                                   /* != 0: a width >= 2^14 */               \
        const uint32_t k = clz_nz(d);                                                                              \
        const uint32_t u = clz_nz(~shl_c((d & low) << 1, k));            /* d & low == low & ~high */              \
        if (lane == (j)) {                                                                                         \
            rec_low = low ^ (lowm & 0x80000000u);                                                                  \
            rec_ku = k | (u << 8);                                                                                 \
        }                                                                                                          \
        lowp = low;                                                                                                \
        s = k + u;                                                                                                 \
        if constexpr (SEEK) wlast = wm1;                                                                           \
    }

    uint32_t b = 0;
    for (uint32_t base = 0; base < n; base += 32, ++b) {
        const uint32_t mine = next;
        const uint32_t nb = base + 32 + lane;
        next = (nb < n) ? __ldg(iv + nb) : 0u;              // prefetch the next 32 intervals
        if constexpr (SEEK) {
            if (base != 0u && base % every == 0u && lane == 0) {
                const uint32_t lowc = shl_c(lowp, s) & 0x7FFFFFFFu;
                const uint32_t sp = min(s, 63u);
                uint32_t *pt = pts + 4u * (base / every - 1u);
                pt[0] = lowc;
                pt[1] = lowc + (uint32_t)((((uint64_t)wlast + 1ull) << sp) - 1ull);
            }
        }
        uint32_t rec_low = 0u, rec_ku = 0u;
        if (n - base >= 32u) {
#pragma unroll
            for (int j = 0; j < 32; ++j) L3C_ENC_STEP(j)
        } else {
            const int cnt = (int)(n - base);
#pragma unroll 1
            for (int j = 0; j < cnt; ++j) L3C_ENC_STEP(j)
        }
        const uint32_t slot = b % ENC_RING;
        if (b >= ENC_RING) mbar_wait(bar0 + 8 * (ENC_RING + slot), (b / ENC_RING - 1) & 1u);    // empty[slot]
        ring[slot][lane] = make_uint2(rec_low, rec_ku);
        mbar_arrive(bar0 + 8 * slot);                                                           // full[slot]
    }
#undef L3C_ENC_STEP

    // termination (torchac.cpp:209-219): one more bit + the owed underflow bits, zero-padded -- i.e. a one-bit
    // record (lane 0) that the emitter meets with pending + 1 owed bits
    const uint32_t low = shl_c(lowp, s) & 0x7FFFFFFFu;
    const uint32_t fin = (low < 0x40000000u) ? 0u : 1u;
    const uint32_t slot = b % ENC_RING;
    if (b >= ENC_RING) mbar_wait(bar0 + 8 * (ENC_RING + slot), (b / ENC_RING - 1) & 1u);
    ring[slot][lane] = lane == 0 ? make_uint2(fin << 31, 1u) : make_uint2(0u, 0u);
    mbar_arrive(bar0 + 8 * slot);
}

// Emitter warp: the batches of 32 records in order, then the termination record; writes the words and out_len.
// SEEK: after the batch that ends before a point, lane 0 writes words 2 and 3 of the point: the code bits the decoder
// has read there, 32 + the sum of k + u over the symbols before it (64 bits: word 2 the low, word 3 the high word), and
// in bit 31 of word 3 whether the last renormalisation shift before it was an underflow shift.  Such a shift
// subtracts 2^30 from the code value before shifting it (torchac.cpp:360), so after it the value is the last 32 code
// bits read with bit 31 flipped; after an "equal MSB" shift it is those bits.  Symbols with no shift leave it as it was.
template <bool SEEK = false>
__device__ __forceinline__ void emit_records(const l3c_enc_stream_t &st, const uint2 (*ring)[32], uint32_t *stage,
                                             uint32_t bar0, int lane, uint32_t *out_len, uint32_t every = 0u,
                                             uint32_t *__restrict__ pts = nullptr) {
    uint64_t bits = 32u;
    uint32_t flip = 0u;
    Emitter em;
    em.stage = stage;
    em.pending = 0u;
    em.sink.out = reinterpret_cast<uint32_t *>(st.out);
    em.sink.cap_words = st.out_cap >> 2;
    em.sink.wpos = 0;
    em.sink.acc = 0;
    em.sink.nacc = 0;
    em.sink.lane = lane;
    const uint32_t n_batches = st.n_sym / 32u + (st.n_sym % 32u != 0u);
    for (uint32_t b = 0; b <= n_batches; ++b) {
        const uint32_t slot = b % ENC_RING;
        mbar_wait(bar0 + 8 * slot, (b / ENC_RING) & 1u);                                        // full[slot]
        const uint2 rec = ring[slot][lane];
        mbar_arrive(bar0 + 8 * (ENC_RING + slot));                                              // empty[slot]
        if (b == n_batches) em.pending += 1u;
        if constexpr (SEEK) {
            if (b < n_batches) {
                const uint32_t k = rec.y & 0xFFu, u = rec.y >> 8;
                bits += __reduce_add_sync(FULL, k + u);
                const uint32_t shifted = __ballot_sync(FULL, k + u != 0u);
                if (shifted) flip = __shfl_sync(FULL, u, 31 - __clz((int)shifted)) != 0u ? 0x80000000u : 0u;
                const uint32_t end = 32u * (b + 1u);
                if (end < st.n_sym && end % every == 0u && lane == 0) {
                    uint32_t *pt = pts + 4u * (end / every - 1u);
                    pt[2] = (uint32_t)bits;
                    pt[3] = (uint32_t)(bits >> 32) | flip;
                }
            }
        }
        em.emit(rec.x, rec.y & 0xFFu, rec.y >> 8);
    }
    BitSink &sink = em.sink;
    // in 64 bits: a stream of 2^32 bytes or more reports 2^32 - 1, which exceeds every out_cap
    const uint64_t total = 4ull * sink.wpos + (uint64_t)((sink.nacc + 7) >> 3);
    if (sink.nacc > 0) {
        const uint32_t w = (uint32_t)(sink.acc << (32 - sink.nacc));
        if (lane == 0 && sink.wpos < sink.cap_words) sink.out[sink.wpos] = __byte_perm(w, 0, 0x0123);
    }
    if (lane == 0) *out_len = (uint32_t)min(total, (uint64_t)0xFFFFFFFFu);
}

// SPC = streams per CTA.  Coding warps are warps 0..SPC-1, emitter warps SPC..2*SPC-1 (the decoders' layout).
template <int SPC>
__global__ void __launch_bounds__(64 * SPC)
ac_encode_kernel(const l3c_enc_stream_t *__restrict__ streams, int n_streams, uint32_t *__restrict__ out_len) {
    __shared__ uint2 s_ring[SPC][ENC_RING][32];
    __shared__ uint32_t s_stage[SPC][STAGE_WORDS];
    __shared__ __align__(8) uint64_t s_bar[SPC][2 * ENC_RING];          // full[0..RING), empty[0..RING)
    const int warp_id = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int sslot = warp_id % SPC;
    const uint32_t bar0 = smem_u32(s_bar[sslot]);
    if (warp_id < SPC && lane == 0) {
#pragma unroll
        for (int i = 0; i < 2 * ENC_RING; ++i) mbar_init(bar0 + 8 * i, 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int sid = blockIdx.x * SPC + sslot;
    if (sid >= n_streams) return;
    const l3c_enc_stream_t st = streams[sid];
    if (warp_id < SPC)
        encode_records(st.intervals, st.n_sym, s_ring[sslot], bar0, lane);
    else
        emit_records(st, s_ring[sslot], s_stage[sslot], bar0, lane, out_len + sid);
}

// ac_encode_kernel that also records the decoder's state every `every` symbols (l3c_ac_encode_streams_seek): the
// same bytes; points[sid] receives 4 words per point (encode_records / emit_records with SEEK)
template <int SPC>
__global__ void __launch_bounds__(64 * SPC)
ac_encode_seek_kernel(const l3c_enc_stream_t *__restrict__ streams, int n_streams, uint32_t *__restrict__ out_len,
                      uint32_t every, uint32_t *const *__restrict__ points) {
    __shared__ uint2 s_ring[SPC][ENC_RING][32];
    __shared__ uint32_t s_stage[SPC][STAGE_WORDS];
    __shared__ __align__(8) uint64_t s_bar[SPC][2 * ENC_RING];
    const int warp_id = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int sslot = warp_id % SPC;
    const uint32_t bar0 = smem_u32(s_bar[sslot]);
    if (warp_id < SPC && lane == 0) {
#pragma unroll
        for (int i = 0; i < 2 * ENC_RING; ++i) mbar_init(bar0 + 8 * i, 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int sid = blockIdx.x * SPC + sslot;
    if (sid >= n_streams) return;
    const l3c_enc_stream_t st = streams[sid];
    uint32_t *pts = points[sid];
    if (warp_id < SPC)
        encode_records<true>(st.intervals, st.n_sym, s_ring[sslot], bar0, lane, every, pts);
    else
        emit_records<true>(st, s_ring[sslot], s_stage[sslot], bar0, lane, out_len + sid, every, pts);
}

// ---------------------------------------------------------------------------------------------
// decoder
// ---------------------------------------------------------------------------------------------

// MSB-first bit reader over a byte stream that may start at ANY address (streams are decoded in
// place from the container): words are fetched from the 4-byte aligned address below the stream and
// the first `8*mis` bits are simply skipped; bytes past the end read as zero (torchac.cpp:109-112).
// Positions never wrap: the window is a 32-bit WORD index (streams are below 2^32 bytes, so words below 2^30 + 1)
// and only bits 0..4 of `pos` are used, so the counter itself may wrap; the bit position is 32 * wbase + (pos & 31),
// formed in 64 bits where it leaves the kernel (save_stream).
struct BitSource {
    const uint32_t *base;
    uint32_t wend;         // words (relative to base) holding at least one byte of the stream: ceil((mis + in_len) / 4)
    uint32_t last_mask;    // the bytes of word wend - 1 that lie inside the stream (big-endian mask)
    uint32_t wbase;        // word index of the upper half of `win`
    uint64_t win;          // words wbase, wbase+1
    uint32_t nextw;        // word wbase+2, ready to use
    uint32_t raw;          // word wbase+3 as loaded (little-endian, unmasked): consumed one refill
                           // later, so its load latency never lands on the coder's serial chain
    uint32_t pos;          // next unread bit: bit (pos & 31) of word wbase; the higher bits are meaningless

    __device__ __forceinline__ uint32_t load_raw(uint32_t i) const { return (i < wend) ? __ldg(base + i) : 0u; }
    __device__ __forceinline__ uint32_t finish(uint32_t w_raw, uint32_t i) const {   // big-endian, zero past the end
        const uint32_t w = __byte_perm(w_raw, 0, 0x0123);
        return w & ((i + 1u < wend) ? FULL : ((i + 1u == wend) ? last_mask : 0u));
    }
    __device__ __forceinline__ uint32_t word(uint32_t i) const { return finish(load_raw(i), i); }
    __device__ __forceinline__ uint32_t open(const uint8_t *in, uint32_t len) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(in);
        const uint32_t mis = (uint32_t)(a & 3u);
        base = reinterpret_cast<const uint32_t *>(a - mis);
        const uint64_t end = (uint64_t)mis + len;          // up to 2^32 + 2: not a 32-bit quantity
        wend = (uint32_t)((end + 3u) >> 2);
        last_mask = (end & 3u) ? (FULL << (8u * (4u - (uint32_t)(end & 3u)))) : FULL;
        return 8u * mis;                                   // bit position of the first code bit
    }
    __device__ __forceinline__ void seek(uint64_t p) {
        wbase = (uint32_t)(p >> 5);
        win = ((uint64_t)word(wbase) << 32) | (uint64_t)word(wbase + 1);
        nextw = word(wbase + 2);
        raw = load_raw(wbase + 3);
        pos = (uint32_t)p;
    }
    __device__ __forceinline__ uint64_t position() const { return 32ull * wbase + (pos & 31u); }
    // the next 32 bits (not consumed)
    __device__ __forceinline__ uint32_t peek32() const { return (uint32_t)((win << (pos & 31u)) >> 32); }
    // (pos & 31) + n <= 63: the window moves by one word exactly when bit 5 of pos flips
    __device__ __forceinline__ void skip(uint32_t n) {     // n <= 32
        const uint32_t p0 = pos;
        pos += n;
        if ((p0 ^ pos) & 32u) {
            win = (win << 32) | (uint64_t)nextw;
            wbase++;
            nextw = finish(raw, wbase + 2);
            raw = load_raw(wbase + 3);
        }
    }
    // same as skip(), written so that it compiles to predicated straight-line code (fast decode loops)
    __device__ __forceinline__ void skip_flat(uint32_t n) {
        const uint32_t p0 = pos;
        pos += n;
        const bool cross = ((p0 ^ pos) & 32u) != 0u;
        const uint32_t fin = finish(raw, wbase + 3);       // becomes word (wbase+1)+2
        const uint32_t idx = wbase + 4u;
        const bool fetch = cross & (idx < wend);
        win = cross ? ((win << 32) | (uint64_t)nextw) : win;
        nextw = cross ? fin : nextw;
        // predicated load straight into `raw` (no select behind it: a select would wait for the load).
        // When nothing is fetched the stale value is harmless: finish() zeroes words past the end.
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.u32 p, %2, 0;\n\t"
            "@p ld.global.nc.u32 %0, [%1];\n\t}"
            : "+r"(raw)
            : "l"(base + idx), "r"((uint32_t)fetch));
        wbase += cross ? 1u : 0u;
    }
    __device__ __forceinline__ uint32_t take(uint32_t n) { // n <= 32; take(0) == 0
        const uint32_t v = shr_c(peek32(), 32u - n);
        skip(n);
        return v;
    }
};

// The saved state (l3c_dec_stream_t.state): low, high, value, then the code bits read, word 3 their low 32 bits.  A
// stream of LONG_STREAM_BYTES or more also keeps their high bits in word 4, so its state takes 5 words; a shorter one
// takes 4.  Every position inside a shorter stream is below 2^31 + 64 bits, so one of 2^32 or more lies far past its
// end, where only zeros are read: such a position is saved as its low 32 bits with bit 31 of word 0 set (a saved low
// never has it, as every renormalisation clears it) and restored as past the end.
constexpr uint32_t LONG_STREAM_BYTES = 1u << 28;
constexpr uint32_t PAST_END = 0x80000000u;

// count of torchac.cpp:327 in the reference's modular 64-bit arithmetic (only needed when the code
// value has left [low, high], i.e. on corrupt or foreign input) -- kept out of line on purpose
__device__ __noinline__ uint32_t foreign_count16(uint32_t value, uint32_t low, uint32_t r) {
    const uint64_t off = (uint64_t)value - (uint64_t)low + 1ull;
    return (uint32_t)(((off * 65536ull - 1ull) / ((uint64_t)r + 1ull)) & 0xFFFFull);
}

// Decoder state: (low, r = high - low, dv = value - low).  Every renormalisation shift maps
// r -> 2r + 1 and dv -> 2dv + next code bit (mod 2^32) and leaves bit 31 of low clear -- for the
// "equal MSB" and the "underflow" shifts alike -- so neither `high`, `value` nor the reference's MSB
// fix-ups (torchac.cpp:345-364) are needed on the serial chain.  Saved/restored as (low, high, value).
struct CoderState {
    uint32_t low, r, dv;
    __device__ __forceinline__ void reset(uint32_t value) {
        low = 0u;
        r = 0xFFFFFFFFu;
        dv = value;
    }
    __device__ __forceinline__ void restore(const uint32_t *st) {
        low = st[0] & ~PAST_END;
        r = st[1] - low;
        dv = st[2] - low;
    }
    __device__ __forceinline__ void save(uint32_t *st) const {
        st[0] = low;
        st[1] = low + r;
        st[2] = low + dv;
    }
    // update() for the speculative fast loop: no branches; returns true when the step needed more
    // than 32 shifts (then the new state is garbage and the caller replays the group with update())
    template <class Source>
    __device__ __forceinline__ bool update_flat(uint32_t c_lo, uint32_t c_hi, Source &src) {
        const uint32_t peek = src.peek32();
        const uint32_t hi16 = (uint32_t)(((uint64_t)r * c_hi + c_hi) >> 16);
        const uint32_t lo16 = (uint32_t)(((uint64_t)r * c_lo + c_lo) >> 16);
        const uint32_t width = hi16 - lo16;
        const uint32_t lo = low + lo16;
        const uint32_t hi = lo + width - 1u;
        const uint32_t d = dv - lo16;
        const uint32_t k = (uint32_t)__clz((int)(lo ^ hi));
        const uint32_t u = clz_nz(~shl_c(shl_c(lo & ~hi, k), 1u));
        const uint32_t s = k + u;
        low = shl_c(shl_c(lo, k), u) & 0x7FFFFFFFu;
        r = shl_c(shl_c(width, k), u) - 1u;
        // (d << s) | (next s code bits): two clamped funnel shifts, the first one overlaps the clz of u
        dv = __funnelshift_lc(shl_c(peek, k), __funnelshift_lc(peek, d, k), u);
        src.skip_flat(s);
        return s > 32u;
    }
    // narrow to [c_lo, c_hi) / 2^16 of the current interval, renormalise, refill  (torchac.cpp:339-364)
    template <class Source>
    __device__ __forceinline__ void update(uint32_t c_lo, uint32_t c_hi, Source &src) {
        const uint32_t hi16 = (uint32_t)(((uint64_t)r * c_hi + c_hi) >> 16);
        const uint32_t lo16 = (uint32_t)(((uint64_t)r * c_lo + c_lo) >> 16);
        const uint32_t width = hi16 - lo16;                 // new high - new low + 1
        const uint32_t lo = low + lo16;
        const uint32_t hi = lo + width - 1u;
        const uint32_t d = dv - lo16;
        const uint32_t k = (uint32_t)__clz((int)(lo ^ hi));
        const uint32_t u = clz_nz(~shl_c(shl_c(lo & ~hi, k), 1u));
        const uint32_t s = k + u;
        if (__builtin_expect(s <= 32u, 1)) {
            const uint32_t bits = src.take(s);
            low = shl_c(lo, s) & 0x7FFFFFFFu;
            r = shl_c(width, s) - 1u;
            dv = shl_c(d, s) | bits;
        } else {
            const uint32_t bk = src.take(k);
            const uint32_t bu = src.take(u);
            low = shl_c(shl_c(lo, k), u) & 0x7FFFFFFFu;
            r = shl_c(shl_c(width, k), u) - 1u;
            dv = shl_c(shl_c(d, k) | bk, u) | bu;
        }
    }
};

// The symbols [first, last) of a stream of n that a launch for [first, first + count) decodes; false when there
// are none.  Symbols below upd_end update the coder state, the stream's final symbol does not (torchac.cpp:335-337).
__device__ __forceinline__ bool chunk_of(uint32_t n, uint32_t first, uint32_t count, uint32_t &last, uint32_t &upd_end) {
    if (first >= n) return false;
    last = (count > n - first) ? n : first + count;
    upd_end = (last == n) ? n - 1u : last;
    return true;
}

// Opens the stream at symbol `first`: at its head when first == 0, else where the previous launch saved its state.
// Returns the bit position of the stream's first code bit (save_stream() needs it).
// SEG (segment mode, l3c_ac_decode_segments): first is 0 and a non-null `state` holds a seek point (low, high, flip,
// bits: low word, high word): the code value is the 32 code bits ending at `bits`, bit 31 flipped by `flip`.
template <bool SEG = false>
__device__ __forceinline__ uint32_t open_stream(const l3c_dec_stream_t &st, uint32_t first, BitSource &src,
                                                CoderState &cs) {
    const uint32_t bit0 = src.open(st.in, st.in_len);
    if (SEG && st.state != nullptr) {
        const uint64_t bits = ((uint64_t)st.state[4] << 32) | st.state[3];
        src.seek(bit0 + bits - 32u);
        const uint32_t value = src.take(32) ^ st.state[2];
        cs.low = st.state[0];
        cs.r = st.state[1] - cs.low;
        cs.dv = value - cs.low;
    } else if (first == 0) {
        src.seek(bit0);
        cs.reset(src.take(32));
    } else {
        cs.restore(st.state);
        const uint64_t hi = (st.in_len >= LONG_STREAM_BYTES) ? st.state[4] : (st.state[0] & PAST_END) ? 1u : 0u;
        src.seek(((hi << 32) | st.state[3]) + bit0);
    }
    return bit0;
}

// one lane per stream (the layout: LONG_STREAM_BYTES above)
__device__ __forceinline__ void save_stream(const l3c_dec_stream_t &st, const CoderState &cs, const BitSource &src,
                                            uint32_t bit0) {
    if (st.state != nullptr) {
        cs.save(st.state);
        const uint64_t bits = src.position() - bit0;
        st.state[3] = (uint32_t)bits;
        if (st.in_len >= LONG_STREAM_BYTES)
            st.state[4] = (uint32_t)(bits >> 32);
        else if (bits >> 32)
            st.state[0] |= PAST_END;
    }
}

__device__ __forceinline__ bool below(uint32_t e, uint32_t r, uint64_t target) {   // e * (r+1) < target
    return ((uint64_t)r * e + e) < target;
}

// One exact, branchy decoding step: the replay of a group the speculative loop gave up on, and the symbols
// outside whole groups.  pk holds this lane's P packed proposals (cdf[m] << 16) | (cdf[m+1] - 1) of the entries
// m = P*lane .. P*lane + P-1; past the alphabet they are 0 or repeat entry L-1's (see v3::ac_decode_kernel), so
// they never change the largest passing proposal.  Returns that winning proposal and updates the state with its
// interval unless `update` is false (the stream's final symbol).
//   reference: count = ((value-low+1)*2^16-1)/span; sym = largest m with cdf[m] <= count, floor 0
//   here:      cdf[m] <= count  <=>  cdf[m]*span < (value-low+1)<<16      (no division)
template <int P>
__device__ __forceinline__ uint32_t exact_step(const uint32_t (&pk)[P], CoderState &cs, BitSource &src, int lane,
                                               bool update) {
    const uint32_t r = cs.r;                                    // span - 1
    const uint32_t dv = cs.dv;
    uint64_t target = ((uint64_t)dv + 1ull) << 16;
    uint32_t r_cmp = r;
    if (__builtin_expect(dv > r, 0)) {
        // value outside [low, high] (corrupt / foreign input): use the reference's truncated count;
        // cdf[m] <= count  <=>  cdf[m] * 1 < count + 1
        target = (uint64_t)foreign_count16(cs.low + dv, cs.low, r) + 1ull;
        r_cmp = 0u;
    }
    uint32_t best = 0u;
#pragma unroll
    for (int j = 0; j < P; ++j) {
        const bool fj = ((lane | j) == 0) || below(pk[j] >> 16, r_cmp, target);
        best = fj ? max(best, pk[j]) : best;
    }
    const uint32_t top = __reduce_max_sync(FULL, best);
    if (update) cs.update(top >> 16, (top & 0xFFFFu) + 1u, src);
    return top;
}

// Writes a group of cnt <= 8 decoded symbols, packed four to a word, to out[0, cnt): as two words when the group
// is whole and out is 4-byte aligned, else byte by byte.  (The byte loop stays rolled: unrolled, the register
// allocation and schedule it brings made both decoders slower, by about 2 % at L = 256 and 10 % at L = 25 on an
// H100 80GB HBM3 at 700 W.)
__device__ __forceinline__ void store_group(uint8_t *out, const uint32_t (&packed)[2], uint32_t cnt) {
    if (cnt == 8u && (reinterpret_cast<uintptr_t>(out) & 3u) == 0u) {
        reinterpret_cast<uint32_t *>(out)[0] = packed[0];
        reinterpret_cast<uint32_t *>(out)[1] = packed[1];
    } else {
        const uint64_t p = ((uint64_t)packed[1] << 32) | packed[0];   // a register, not a local-memory array
#pragma unroll 1
        for (uint32_t d = 0; d < cnt; ++d) out[d] = (uint8_t)(p >> (8 * d));
    }
}

// ---------------------------------------------------------------------------------------------
// decoder, alphabets of at most 32 symbols (bottleneck and uniform-prior streams): one CDF entry per
// lane, one compare and one max-reduction.  Groups of 8 symbols run as straight-line speculative code
// (see v3::ac_decode_kernel); a group that trips the sticky flag is replayed with exact_step().
// ---------------------------------------------------------------------------------------------
// SEG: every descriptor is a segment (l3c_ac_decode_segments), decoded whole from its seek point
template <bool SEG = false>
__global__ void __launch_bounds__(32)
ac_decode32_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, int L,
                   uint32_t first, uint32_t count) {
    constexpr int D = 8;   // symbols per group = row prefetch distance
    const int sid = blockIdx.x;
    if (sid >= n_streams) return;
    const int lane = threadIdx.x & 31;
    const l3c_dec_stream_t st = streams[sid];
    uint32_t last, upd_end;
    if (!chunk_of(st.n_sym, first, count, last, upd_end)) return;

    BitSource src;
    CoderState cs;
    const uint32_t bit0 = open_stream<SEG>(st, first, src, cs);

    const uint16_t *__restrict__ table = st.table;
    const int64_t pitch = st.row_pitch;
    uint8_t *__restrict__ sym_out = st.sym_out;
    const bool in_row = lane < L;

    // the speculative groups: whole groups of D, never the stream's final symbol
    const uint32_t main_end = first + ((upd_end - first) / D) * D;

    // lane l keeps entry l as the packed proposal (cdf[l] << 16) | (cdf[l+1] - 1) (2^16 after the last
    // entry), built when the row arrives: rows are sorted, so the warp-max over the passing proposals
    // is the decoded symbol's and carries both interval bounds -- one REDUX instead of
    // ballot -> popc -> two shuffles on the serial chain (the symbol index itself is off the chain).
    // (the packing is done when a row is used, not when it is loaded: a shuffle right behind the load
    // would put the HBM latency of every row on the critical path)
    auto pack_row = [&](uint32_t v) -> uint32_t {
        uint32_t nx = __shfl_down_sync(FULL, v, 1);
        if (lane + 1 >= L) nx = 0x10000u;
        return in_row ? ((v << 16) | ((nx - 1u) & 0xFFFFu)) : 0u;
    };
    // symbol i on the exact path; the symbol is the number of the row's proposals up to the winner, minus 1
    auto exact = [&](uint32_t i) {
        const uint32_t pk[1] = {pack_row((uint32_t)__ldg(table + (int64_t)i * pitch + lane))};
        const uint32_t top = exact_step(pk, cs, src, lane, i < upd_end);
        const int sym = __popc(__ballot_sync(FULL, in_row && pk[0] <= top)) - 1;
        if (lane == 0) sym_out[i] = (uint8_t)sym;
    };
    // rows are fetched two groups ahead: a group's rows are packed at its start, so they must have been
    // requested at least a whole group (~1.5 us) earlier for HBM latency to stay hidden
    uint32_t ring[D], ahead[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const uint32_t i = first + d;
        ring[d] = (i < main_end) ? (uint32_t)__ldg(table + (int64_t)i * pitch + lane) : 0u;
        ahead[d] = (i + D < main_end) ? (uint32_t)__ldg(table + (int64_t)(i + D) * pitch + lane) : 0u;
    }
    uint32_t base = first;
    for (; base < main_end; base += D) {
        {
            const CoderState cs0 = cs;
            const BitSource src0 = src;
            bool bad = false;
            uint32_t packed[D / 4];
            uint32_t prop[D];
#pragma unroll
            for (int d = 0; d < D; ++d) prop[d] = pack_row(ring[d]);   // off the serial chain
#pragma unroll
            for (int d = 0; d < D; ++d) {
                const uint32_t i = base + d;
                const uint32_t pk = prop[d];
                ring[d] = ahead[d];
                // (clamped, not predicated: a conditional load into the array costs a select that waits for it)
                ahead[d] = (uint32_t)__ldg(table + (int64_t)min(i + 2 * D, main_end - 1u) * pitch + lane);
                const uint32_t r = cs.r, dv = cs.dv;
                const uint32_t span = r + 1u;                        // 2^32 wraps to 0: replay (stream start)
                bad |= (dv > r) || (span == 0u);
                // cdf[m] <= count  <=>  mulhi(cdf[m] << 16, span) <= dv
                const bool f = (lane == 0) || (in_row && __umulhi(pk & 0xFFFF0000u, span) <= dv);
                const uint32_t top = __reduce_max_sync(FULL, f ? pk : 0u);
                const int nt = __popc(__ballot_sync(FULL, f));       // symbol + 1 (not on the chain)
                bad |= cs.update_flat(top >> 16, (top & 0xFFFFu) + 1u, src);
                if ((d & 3) == 0) packed[d >> 2] = 0u;
                packed[d >> 2] |= (uint32_t)(nt - 1) << (8 * (d & 3));
            }
            if (__builtin_expect(!bad, 1)) {
                if (lane == 0) store_group(sym_out + base, packed, D);
                continue;
            }
            cs = cs0;                 // replay this group exactly (the ring already holds the next group's rows)
            src = src0;
        }
#pragma unroll 1
        for (int d = 0; d < D; ++d) exact(base + d);
    }
    // tail (< D symbols, may contain the stream's final symbol)
#pragma unroll 1
    for (uint32_t i = base; i < last; ++i) exact(i);

    if (!SEG && lane == 0) save_stream(st, cs, src, bit0);
}

// ---------------------------------------------------------------------------------------------
// decoder, alphabets of 33 to 256 symbols (the RGB streams have 256): CTA = decoder warp + helper warp
// per stream; rows are read as 256 entries whatever L is
//
// A single warp issues one dependent instruction every ~4-5 cycles, so the serial rate of the coder
// is set by the number of instructions the decoding warp executes per symbol.  Everything that does
// not depend on the coder state is therefore moved to a second warp (another scheduler of the SM):
//   helper warp : prefetches CDF rows from HBM one group (8 symbols) ahead, turns every entry m into
//                 the packed proposal (cdf[m] << 16) | (cdf[m+1] - 1) and stores the row in a shared
//                 memory ring; later turns the decoder's winning proposals into symbol indices
//                 (number of proposals <= winner, minus 1) and writes them out.
//   decoder warp: per lane eight compares  mulhi(cdf[m] << 16, span) <= value - low  (no division: this
//                 is cdf[m] <= count of torchac.cpp:327), ONE warp max-reduction (rows are sorted,
//                 so the last passing proposal is the largest) that yields both interval bounds,
//                 then the update / clz renormalisation / funnel-shift refill on (low, r, dv).
//                 Groups of 8 symbols run as straight-line SPECULATIVE code: the two events that
//                 cannot occur on a valid stream (code value outside [low, high], > 32 shifts) and
//                 the 2^32 span of a stream's first symbol only set a sticky flag, after which the
//                 group is replayed from a checkpoint by the exact, branchy path.
// Hand-over by two mbarrier pairs (full/empty per group of 8 ring slots).
// ---------------------------------------------------------------------------------------------
namespace v3 {

constexpr int G = 8;            // symbols per group
constexpr int R = 2 * G;        // ring slots


// SPC = streams per CTA.  Decoder warps are warps 0..SPC-1, helper warps SPC..2*SPC-1: with SPC = 4 the
// decoder and the helper of a stream sit on the same SM sub-partition (warp id mod 4) and every scheduler
// serves exactly one latency-bound decoder warp -- a CTA of 4 streams fills one SM, so a batch of 48
// streams needs 12 SMs and several batches can be decoded side by side.
constexpr int RING_BYTES = R * 2 * 32 * 16;           // 16 KB of proposals per stream
constexpr int STREAM_SMEM = RING_BYTES + 128;         // + tops[R] (64 B) + 4 mbarriers (32 B), 16-byte aligned

// one speculative group of G symbols (decoder warp).  FULL2: the group starts with a span of exactly 2^32.
template <bool FULL2>
__device__ __forceinline__ bool spec_group(CoderState &cs, BitSource &src, const uint4 *slot, uint32_t *tops, int lane) {
    bool bad = false;
    uint4 a = slot[0], b = slot[32];
#pragma unroll 1
    for (int d = 0; d < G; ++d) {
        const uint4 *nslot = slot + ((d + 1) & (G - 1)) * 64;         // next symbol's proposals
        const uint4 na = nslot[0], nb = nslot[32];
        const uint32_t r = cs.r, dv = cs.dv;
        const uint32_t span = r + 1u;                                 // 2^32 wraps to 0
        bad |= (dv > r) || ((span == 0u) != FULL2);
        // cdf[m] <= count  <=>  cdf[m] * span < (dv + 1) << 16  <=>  mulhi(cdf[m] << 16, span) <= dv
        const uint32_t pk[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        bool f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            f[j] = (FULL2 ? (pk[j] & 0xFFFF0000u) : __umulhi(pk[j] & 0xFFFF0000u, span)) <= dv;
        f[0] = f[0] || (lane == 0);                                   // symbol 0 is the floor
        // rows are sorted: the last passing proposal is the numerically largest
        const uint32_t m01 = f[1] ? pk[1] : (f[0] ? pk[0] : 0u);
        const uint32_t m23 = f[3] ? pk[3] : (f[2] ? pk[2] : 0u);
        const uint32_t m45 = f[5] ? pk[5] : (f[4] ? pk[4] : 0u);
        const uint32_t m67 = f[7] ? pk[7] : (f[6] ? pk[6] : 0u);
        const uint32_t top = __reduce_max_sync(FULL, max(max(m01, m23), max(m45, m67)));
        if (lane == 0) tops[d] = top;
        bad |= cs.update_flat(top >> 16, (top & 0xFFFFu) + 1u, src);
        a = na;
        b = nb;
    }
    return bad;
}

// FULLROW: L = 256.  Otherwise (33 <= L <= 255) only the helper warp differs, and nothing it does depends on what
// the row holds past entry L-1:
//   * entry L-1's upper bound is 2^16;
//   * entries m >= L propose 0, which passes every compare but never exceeds entry 0's proposal (that always
//     passes) -- except entry L when it shares a pair of spec_group's select tree with entry L-1 (odd L): a 0 there
//     would pass and hide entry L-1, so it repeats entry L-1's proposal, which passes exactly when that one does;
//   * only entries m < L count towards the symbol index.
// SEG: segment mode (see ac_decode32_kernel)
template <bool FULLROW, int SPC, bool SEG = false>
__global__ void __launch_bounds__(64 * SPC)
ac_decode_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, int L, uint32_t first, uint32_t count) {
    extern __shared__ __align__(16) uint8_t dec_smem[];
    const int warp_id = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int sslot = warp_id % SPC;                    // stream slot inside the CTA
    const int warp = warp_id / SPC;                     // 0 = decoder, 1 = helper
    uint8_t *mine = dec_smem + sslot * STREAM_SMEM;
    uint4 (*ring)[2][32] = reinterpret_cast<uint4 (*)[2][32]>(mine);          // proposals: [slot][half][lane]
    uint32_t *tops = reinterpret_cast<uint32_t *>(mine + RING_BYTES);         // winning proposal per slot (decoder -> helper)
    uint64_t *bars = reinterpret_cast<uint64_t *>(mine + RING_BYTES + 64);    // full[0..1], empty[0..1]

    const uint32_t bar0 = smem_u32(bars);
    if (warp == 0 && lane == 0) {
        mbar_init(bar0 + 0, 32);
        mbar_init(bar0 + 8, 32);
        mbar_init(bar0 + 16, 32);
        mbar_init(bar0 + 24, 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int sid = blockIdx.x * SPC + sslot;
    if (sid >= n_streams) return;
    const l3c_dec_stream_t st = streams[sid];
    uint32_t last, upd_end;
    if (!chunk_of(st.n_sym, first, count, last, upd_end)) return;
    const uint32_t n_groups = (last - first + G - 1) / G;

    if (warp == 1) {
        // ============================ helper warp ============================
        const uint16_t *__restrict__ table = st.table;
        const int64_t pitch = st.row_pitch;
        uint8_t *__restrict__ sym_out = st.sym_out;
        uint4 nxt[G];
#pragma unroll
        for (int d = 0; d < G; ++d) {
            const uint32_t i = first + d;
            if (i < last) nxt[d] = __ldg(reinterpret_cast<const uint4 *>(table + (int64_t)i * pitch) + lane);
        }
        for (uint32_t gi = 0; gi < n_groups + 2; ++gi) {
            const uint32_t g = gi & 1u;
            uint4 cur[G];
#pragma unroll
            for (int d = 0; d < G; ++d) cur[d] = nxt[d];
            if (gi + 1 < n_groups) {
#pragma unroll
                for (int d = 0; d < G; ++d) {
                    const uint32_t i = first + (gi + 1) * G + d;
                    if (i < last) nxt[d] = __ldg(reinterpret_cast<const uint4 *>(table + (int64_t)i * pitch) + lane);
                }
            }
            if (gi >= 2) {
                // the decoder is done with the rows that live in this half of the ring: turn its
                // winning proposals into symbols, then the slots may be overwritten
                mbar_wait(bar0 + 16 + 8 * g, ((gi >> 1) - 1) & 1u);
                const uint32_t ibase = first + (gi - 2) * G;
                uint32_t packed[2] = {0u, 0u};
#pragma unroll
                for (int d = 0; d < G; ++d) {
                    if (ibase + d < last) {
                        const uint32_t top = tops[g * G + d];
                        const uint4 a = ring[g * G + d][0][lane];
                        const uint4 b = ring[g * G + d][1][lane];
                        const uint32_t pk[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                        int c = 0;
#pragma unroll
                        for (int j = 0; j < 8; ++j) c += (pk[j] <= top && (FULLROW || 8 * lane + j < L)) ? 1 : 0;
                        int tot = __reduce_add_sync(FULL, c);
                        tot = tot > 0 ? tot - 1 : 0;
                        packed[d >> 2] |= (uint32_t)tot << (8 * (d & 3));
                    }
                }
                if (lane == 0) store_group(sym_out + ibase, packed, min(last - ibase, (uint32_t)G));
                __syncwarp();
            }
            if (gi < n_groups) {
#pragma unroll
                for (int d = 0; d < G; ++d) {
                    const uint4 v = cur[d];
                    uint32_t nx = __shfl_down_sync(FULL, v.x, 1);
                    if (lane == 31) nx = 0u;                                  // row end -> upper bound 2^16
                    // proposal of entry m = 8 * lane + j: (cdf[m] << 16) | ((cdf[m+1] - 1) & 0xFFFF)
                    uint32_t p[8] = {(v.x << 16) | (((v.x >> 16) - 1u) & 0xFFFFu),
                                     (v.x & 0xFFFF0000u) | (((v.y & 0xFFFFu) - 1u) & 0xFFFFu),
                                     (v.y << 16) | (((v.y >> 16) - 1u) & 0xFFFFu),
                                     (v.y & 0xFFFF0000u) | (((v.z & 0xFFFFu) - 1u) & 0xFFFFu),
                                     (v.z << 16) | (((v.z >> 16) - 1u) & 0xFFFFu),
                                     (v.z & 0xFFFF0000u) | (((v.w & 0xFFFFu) - 1u) & 0xFFFFu),
                                     (v.w << 16) | (((v.w >> 16) - 1u) & 0xFFFFu),
                                     (v.w & 0xFFFF0000u) | (((nx & 0xFFFFu) - 1u) & 0xFFFFu)};
                    if (!FULLROW) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int m = 8 * lane + j;
                            if (m == L - 1) p[j] |= 0xFFFFu;
                            else if (m >= L) p[j] = (m == L && (j & 1)) ? p[j - 1] : 0u;
                        }
                    }
                    ring[g * G + d][0][lane] = make_uint4(p[0], p[1], p[2], p[3]);
                    ring[g * G + d][1][lane] = make_uint4(p[4], p[5], p[6], p[7]);
                }
                mbar_arrive(bar0 + 8 * g);                                    // full[g]
            }
        }
        return;
    }

    // ============================ decoder warp ============================
    BitSource src;
    CoderState cs;
    const uint32_t bit0 = open_stream<SEG>(st, first, src, cs);
    for (uint32_t gi = 0; gi < n_groups; ++gi) {
        const uint32_t g = gi & 1u;
        mbar_wait(bar0 + 8 * g, (gi >> 1) & 1u);                              // full[g]
        const uint32_t ibase = first + gi * G;
        bool replay = ibase + G > upd_end;                                    // ragged / final group
        if (!replay) {
            // Speculative fast path: straight-line code, no per-symbol checks.  The two things that
            // cannot happen on a valid stream -- code value outside [low, high], more than 32
            // renormalisation shifts -- only set a sticky flag; the group is then replayed exactly.
            const CoderState cs0 = cs;
            const BitSource src0 = src;
            const uint4 *slot = &ring[g * G][0][lane];
            // A span of exactly 2^32 (r + 1 wraps to 0) is the state of a stream's first symbol -- and of EVERY
            // symbol when all probabilities are the same power of two (the uniform prior with L = 256: each
            // symbol narrows the interval to 2^24 and renormalises by exactly 8 bits; such streams used to replay
            // every group: 495 ns per symbol).  mulhi(x, 2^32) = x: those groups run a second copy of the loop
            // without the multiply; a group that mixes the two kinds of state sets `bad` and is replayed.
            const bool bad = (cs.r == 0xFFFFFFFFu) ? spec_group<true>(cs, src, slot, tops + g * G, lane)
                                                    : spec_group<false>(cs, src, slot, tops + g * G, lane);
            if (__builtin_expect(bad, 0)) {
                cs = cs0;
                src = src0;
                replay = true;
            }
        }
        if (replay) {
#pragma unroll 1
            for (int d = 0; d < G; ++d) {
                const uint32_t i = ibase + d;
                if (i >= last) break;
                const uint4 a = ring[g * G + d][0][lane];
                const uint4 b = ring[g * G + d][1][lane];
                const uint32_t pk[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                const uint32_t top = exact_step(pk, cs, src, lane, i < upd_end);
                if (lane == 0) tops[g * G + d] = top;
            }
        }
        __syncwarp();
        mbar_arrive(bar0 + 16 + 8 * g);                                       // empty[g]
    }
    if (!SEG && lane == 0) save_stream(st, cs, src, bit0);
}

}  // namespace v3

// ---------------------------------------------------------------------------------------------
// decoder, RGB streams from coarse rows (L = 256; dmll_math.cuh: per symbol the 30 mixture parameters and the
// coarse entries cdf[8 i]): v3's CTA layout (decoder warp + helper warp per stream, SPC streams per CTA), its
// mbarrier ring and its speculative groups of 8, with a two-level search:
//   helper warp : prefetches each symbol's record one group ahead and writes it into the ring: the parameters
//                 (32 words), the coarse proposals (cdf[8 l] << 16) | (cdf[8 l + 8] - 1), one per lane (2^16 above
//                 cdf[248]), and in the padding word LIN_WORD the linear-bracket mask: bit l set when every term
//                 is saturated on the same side at both ends of bracket l (dmll_math.cuh: mixture_linear), i.e.
//                 cdf[8 l + e] = cdf[8 l] + e.  Narrow components make most brackets of a record linear.
//   decoder warp: level 1 -- lane l compares coarse entry 8 l, one REDUX.MAX gives the bracket's bounds cdf[8 j]
//                 and cdf[8 j + 8], a ballot gives j; level 2 -- lane e < 8 proposes cdf[8 j + e]: cdf[8 j] + e in a
//                 linear bracket, else evaluated term-parallel on 28 lanes (bracket_entry_terms: mixture_cdf_u16's
//                 operations in its order, so the full row's integers); one compare each, and two reductions give
//                 the largest passing entry and the smallest failing one (or cdf[8 j + 8]): the symbol's interval.
// The rows are sorted, so the largest passing coarse entry brackets the largest passing entry of the full row:
// every symbol and every interval is the full-row decoder's.  The exact path (replayed groups, ragged tails, the
// final symbol, corrupt input) runs both levels as exact_step().  The decoder writes the symbols itself.
// ---------------------------------------------------------------------------------------------
namespace coarse {

using v3::G;
using v3::R;

constexpr int SLOT_WORDS = COARSE_PARAM_WORDS + COARSE_N;     // parameters, then the coarse proposals
constexpr int RING_BYTES = R * SLOT_WORDS * 4;                 // 4 KB per stream
constexpr int STREAM_SMEM = RING_BYTES + 32;                   // + 4 mbarriers
constexpr int TG_BYTES = 256 * 4;                              // the targets, shared by the CTA's streams
constexpr float SCALE = (float)(65536 - 256);

inline size_t smem_bytes(int spc) { return (size_t)TG_BYTES + (size_t)spc * STREAM_SMEM; }

constexpr int K = 10;
constexpr int LIN_WORD = 3 * K;          // ring slot word 30 (record padding): the linear-bracket mask

// Entry cdf[8 j + (lane & 7)] of a bracket that is not linear, term-parallel: lane e + 8 q (e = lane & 7) evaluates
// terms q, q + 4, q + 8 (< K) of entry 8 j + e with mixture_term()'s operations, and lane e gathers the K factors by
// shuffles and accumulates them in term order, exactly as mixture_cdf_u16() does.  A term with u >= SAT_HI adds
// nothing; it travels as the factor -1, which no evaluated factor can be (1, a reciprocal of a number >= 1, or
// NaN, for which `< 0` is false) -- a zero factor would not do: fma(NaN, 0, acc) is not acc.  3 MUFU pairs per
// lane instead of 10.  Valid on lanes 1..7 (lane 0 computes cdf[8 j] itself); warp-collective.
__device__ __forceinline__ uint32_t bracket_entry_terms(const float *slot, const float *s_tg, uint32_t j, int lane) {
    const int e = lane & (COARSE_STEP - 1), q = lane >> 3;
    const int m = COARSE_STEP * (int)j + e;
    const float t = s_tg[m];
    float f[3];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
        const int k = (q + 4 * s < K) ? q + 4 * s : q;             // lanes 16..31 own 2 terms; the third is unused
        const float u = __fmul_rn(__fsub_rn(t, slot[K + k]), slot[2 * K + k]);
        const float sig = (u <= SAT_LO) ? 1.0f : sigmoid_from_log2(u);
        f[s] = (u >= SAT_HI) ? -1.0f : sig;
    }
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float x = __shfl_sync(FULL, f[k >> 2], e + COARSE_STEP * (k & 3));
        acc = (x < 0.0f) ? acc : __fmaf_rn(slot[k], x, acc);
    }
    return (uint32_t)(__float2int_rn(__fmul_rn(acc, SCALE)) + m) & 0xFFFFu;
}

// cdf[8 j + lane] on lanes 0..7 (lane 0: cdf[8 j], the bracket's coarse entry top1 >> 16); other lanes: unused.
// lin: the slot's linear-bracket mask.  A linear bracket needs no evaluation: its entries are cdf[8 j] + lane.
__device__ __forceinline__ uint32_t bracket_entry(const uint32_t *slot, uint32_t lin, const float *s_tg, uint32_t j,
                                                  uint32_t top1, int lane) {
    const uint32_t head = top1 >> 16;
    uint32_t v = (head + (uint32_t)lane) & 0xFFFFu;
    if (!((lin >> j) & 1u)) {          // warp-uniform; a select would pay for the evaluation on every symbol
        v = bracket_entry_terms(reinterpret_cast<const float *>(slot), s_tg, j, lane);
        v = (lane == 0) ? head : v;
    }
    return v;
}

// one exact step of both levels; returns the symbol
__device__ __forceinline__ uint32_t exact_symbol(const uint32_t *slot, const float *s_tg, CoderState &cs,
                                                 BitSource &src, int lane, bool update) {
    const uint32_t lin = slot[LIN_WORD];
    const uint32_t pk1[1] = {slot[COARSE_PARAM_WORDS + lane]};
    const uint32_t top1 = exact_step(pk1, cs, src, lane, false);
    const uint32_t j = (uint32_t)__popc(__ballot_sync(FULL, pk1[0] <= top1)) - 1u;
    const uint32_t v = bracket_entry(slot, lin, s_tg, j, top1, lane);
    uint32_t nx = __shfl_down_sync(FULL, v, 1);
    if (lane == COARSE_STEP - 1) nx = (top1 & 0xFFFFu) + 1u;                 // cdf[8 j + 8]
    const uint32_t pk2[1] = {lane < COARSE_STEP ? ((v << 16) | ((nx - 1u) & 0xFFFFu)) : 0u};
    const uint32_t top2 = exact_step(pk2, cs, src, lane, update);
    return COARSE_STEP * j + (uint32_t)__popc(__ballot_sync(FULL, lane < COARSE_STEP && pk2[0] <= top2)) - 1u;
}

// one speculative group of G symbols (see v3::spec_group; FULL2: the group starts with a span of exactly 2^32)
template <bool FULL2>
__device__ __forceinline__ bool spec_group(CoderState &cs, BitSource &src, const uint32_t *ring, const float *s_tg,
                                           int lane, uint32_t (&packed)[2]) {
    bool bad = false;
    uint32_t cp = ring[COARSE_PARAM_WORDS + lane];
#pragma unroll 1
    for (int d = 0; d < G; ++d) {
        const uint32_t *slot = ring + d * SLOT_WORDS;
        const uint32_t ncp = ring[((d + 1) & (G - 1)) * SLOT_WORDS + COARSE_PARAM_WORDS + lane];
        const uint32_t lin = slot[LIN_WORD];                                  // off the chain until j is known
        const uint32_t r = cs.r, dv = cs.dv;
        const uint32_t span = r + 1u;
        bad |= (dv > r) || ((span == 0u) != FULL2);
        auto passes = [&](uint32_t x) {   // cdf <= count  <=>  mulhi(cdf << 16, span) <= dv
            return (FULL2 ? (x & 0xFFFF0000u) : __umulhi(x & 0xFFFF0000u, span)) <= dv;
        };
        // level 1: the bracket
        const bool f1 = (lane == 0) || passes(cp);
        const uint32_t top1 = __reduce_max_sync(FULL, f1 ? cp : 0u);
        const uint32_t j = 31u - (uint32_t)__clz((int)__ballot_sync(FULL, f1));
        // level 2: the entry inside it
        const uint32_t v = bracket_entry(slot, lin, s_tg, j, top1, lane);
        const bool in = lane < COARSE_STEP;
        const bool f2 = (lane == 0) || (in && passes(v << 16));
        const uint32_t lo = __reduce_max_sync(FULL, f2 ? v : 0u);
        const uint32_t hi = __reduce_min_sync(FULL, (in && !f2) ? v : (top1 & 0xFFFFu) + 1u);
        const uint32_t sym = COARSE_STEP * j + (uint32_t)__popc(__ballot_sync(FULL, f2)) - 1u;   // off the chain
        bad |= cs.update_flat(lo, hi, src);
        const uint32_t sh = sym << (8 * (d & 3));
        packed[0] |= (d < 4) ? sh : 0u;
        packed[1] |= (d < 4) ? 0u : sh;
        cp = ncp;
    }
    return bad;
}

// streams: row_pitch >= COARSE_REC_U16 (uint16), table 4-byte aligned; targets_dev: the 256 RGB bin targets
// SEG: segment mode (see ac_decode32_kernel)
template <int SPC, bool SEG = false>
__global__ void __launch_bounds__(64 * SPC, 1)
ac_decode_coarse_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, const float *__restrict__ targets,
                        uint32_t first, uint32_t count) {
    extern __shared__ __align__(16) uint8_t dec_smem[];
    const int warp_id = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int sslot = warp_id % SPC;
    const int warp = warp_id / SPC;                     // 0 = decoder, 1 = helper
    float *s_tg = reinterpret_cast<float *>(dec_smem);
    uint8_t *mine = dec_smem + TG_BYTES + sslot * STREAM_SMEM;
    uint32_t *ring = reinterpret_cast<uint32_t *>(mine);                     // [slot][SLOT_WORDS]
    const uint32_t bar0 = smem_u32(mine + RING_BYTES);                      // full[0..1], empty[0..1]
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_tg[i] = __ldg(targets + i);
    if (warp == 0 && lane == 0) {
        mbar_init(bar0 + 0, 32);
        mbar_init(bar0 + 8, 32);
        mbar_init(bar0 + 16, 32);
        mbar_init(bar0 + 24, 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int sid = blockIdx.x * SPC + sslot;
    if (sid >= n_streams) return;
    const l3c_dec_stream_t st = streams[sid];
    uint32_t last, upd_end;
    if (!chunk_of(st.n_sym, first, count, last, upd_end)) return;
    const uint32_t n_groups = (last - first + G - 1) / G;

    if (warp == 1) {
        // ============================ helper warp ============================
        const uint16_t *__restrict__ table = st.table;
        const int64_t pitch = st.row_pitch;
        const float t_first = s_tg[COARSE_STEP * lane], t_last = s_tg[COARSE_STEP * lane + COARSE_STEP - 1];
        uint32_t nw[G], nc[G];
        auto fetch = [&](uint32_t gi) {
#pragma unroll
            for (int d = 0; d < G; ++d) {
                const uint32_t i = first + gi * G + d;
                if (i < last) {
                    const uint16_t *rec = table + (int64_t)i * pitch;
                    nw[d] = __ldg(reinterpret_cast<const uint32_t *>(rec) + lane);
                    nc[d] = __ldg(rec + 2 * COARSE_PARAM_WORDS + lane);
                } else {
                    nw[d] = nc[d] = 0u;
                }
            }
        };
        fetch(0);
        for (uint32_t gi = 0; gi < n_groups; ++gi) {
            const uint32_t g = gi & 1u;
            uint32_t cw[G], cc[G];
#pragma unroll
            for (int d = 0; d < G; ++d) {
                cw[d] = nw[d];
                cc[d] = nc[d];
            }
            if (gi + 1 < n_groups) fetch(gi + 1);
            if (gi >= 2) mbar_wait(bar0 + 16 + 8 * g, ((gi >> 1) - 1) & 1u);   // the decoder is done with this half
#pragma unroll
            for (int d = 0; d < G; ++d) {
                uint32_t *slot = ring + (g * G + d) * SLOT_WORDS;
                uint32_t nx = __shfl_down_sync(FULL, cc[d], 1);
                if (lane == 31) nx = 0x10000u;                                   // cdf[256]
                slot[lane] = cw[d];
                slot[COARSE_PARAM_WORDS + lane] = (cc[d] << 16) | ((nx - 1u) & 0xFFFFu);
            }
            __syncwarp();
            // bit l of word LIN_WORD: bracket l is linear (mixture_linear() at its first and last entry)
#pragma unroll 1
            for (int d = 0; d < G; ++d) {
                uint32_t *slot = ring + (g * G + d) * SLOT_WORDS;
                const float *w = reinterpret_cast<const float *>(slot);
                const uint32_t lin = __ballot_sync(FULL, mixture_linear<K>(w + K, w + 2 * K, t_first, t_last));
                if (lane == 0) slot[LIN_WORD] = lin;
            }
            mbar_arrive(bar0 + 8 * g);                                           // full[g]
        }
        return;
    }

    // ============================ decoder warp ============================
    BitSource src;
    CoderState cs;
    const uint32_t bit0 = open_stream<SEG>(st, first, src, cs);
    uint8_t *__restrict__ sym_out = st.sym_out;
    for (uint32_t gi = 0; gi < n_groups; ++gi) {
        const uint32_t g = gi & 1u;
        mbar_wait(bar0 + 8 * g, (gi >> 1) & 1u);                                 // full[g]
        const uint32_t ibase = first + gi * G;
        const uint32_t *slots = ring + g * G * SLOT_WORDS;
        bool replay = ibase + G > upd_end;                                       // ragged / final group
        uint32_t packed[2] = {0u, 0u};
        if (!replay) {
            const CoderState cs0 = cs;
            const BitSource src0 = src;
            const bool bad = (cs.r == 0xFFFFFFFFu) ? spec_group<true>(cs, src, slots, s_tg, lane, packed)
                                                    : spec_group<false>(cs, src, slots, s_tg, lane, packed);
            if (__builtin_expect(bad, 0)) {
                cs = cs0;
                src = src0;
                packed[0] = packed[1] = 0u;
                replay = true;
            }
        }
        if (replay) {
#pragma unroll 1
            for (int d = 0; d < G; ++d) {
                const uint32_t i = ibase + d;
                if (i >= last) break;
                const uint32_t sym = exact_symbol(slots + d * SLOT_WORDS, s_tg, cs, src, lane, i < upd_end);
                const uint32_t sh = sym << (8 * (d & 3));
                packed[0] |= (d < 4) ? sh : 0u;
                packed[1] |= (d < 4) ? 0u : sh;
            }
        }
        __syncwarp();
        mbar_arrive(bar0 + 16 + 8 * g);                                          // empty[g]
        if (lane == 0) store_group(sym_out + ibase, packed, min(last - ibase, (uint32_t)G));
    }
    if (!SEG && lane == 0) save_stream(st, cs, src, bit0);
}

}  // namespace coarse

// ---------------------------------------------------------------------------------------------
// decoder, alphabets of 257 to 32768 symbols (reached through the drop-in torchac API): CTA = decoder warp +
// helper warp, one stream per CTA.  A row no longer fits the warp's registers, so it is staged whole in shared
// memory and searched in two levels, each one exact_step() (floor rule, foreign count) over at most 8 proposals
// per lane:
//   helper warp : copies every row into a ring of shared-memory slots with one cp.async.bulk (its mbarrier
//                 completes on the transaction bytes), up to ring_n - 1 rows ahead of the decoder; once a row has
//                 landed it writes the row's 256 bucket heads (cdf[j*s] << 16) | j, s = ceil(L/256), 8 per lane
//                 in v3's ring layout (heads of buckets past the row propose 0, which never wins).
//   decoder warp: level 1: the largest passing head gives the bucket j (rows are sorted, so the head of bucket j+1
//                 fails whenever it exists); level 2: entries m0 + lane + 32t of bucket j (m0 = j*s, s <= 128)
//                 propose (cdf[m] << 16) | (cdf[m+1] - 1), 2^16 above entry L-1; entry m0 always passes (floor
//                 0 for j = 0, its head passed otherwise), the largest passing proposal carries the interval, and
//                 the number of proposals up to it gives the symbol.  No speculation: every symbol runs the exact
//                 step, so corrupt input needs no replay.
// Symbols are written as uint16.
// ---------------------------------------------------------------------------------------------
namespace wide {

constexpr int MAX_RING = 8;                   // row slots at most
constexpr int BAR_BYTES = 3 * MAX_RING * 8;   // tx / full / empty mbarrier per slot
constexpr int HEAD_BYTES = 256 * 4;           // 256 packed bucket heads per slot

__host__ __device__ inline uint32_t row_bytes(int L) { return (uint32_t)((L + 7) & ~7) * 2u; }
inline size_t smem_bytes(int ring_n, int L) { return BAR_BYTES + (size_t)ring_n * (HEAD_BYTES + row_bytes(L)); }

// one row, global -> shared, completing `bar`'s current phase on its bytes (16-byte aligned, multiple of 16)
__device__ __forceinline__ void stage_row(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

__global__ void __launch_bounds__(64)
ac_decode_wide_kernel(const l3c_dec_stream_t *__restrict__ streams, int L, int ring_n, uint32_t first,
                      uint32_t count) {
    extern __shared__ __align__(16) uint8_t dec_smem[];
    const int warp = threadIdx.x >> 5;                 // 0 = decoder, 1 = helper
    const int lane = threadIdx.x & 31;
    const uint32_t bars = smem_u32(dec_smem);
    const uint32_t rb = row_bytes(L);
    uint4 (*heads)[2][32] = reinterpret_cast<uint4 (*)[2][32]>(dec_smem + BAR_BYTES);          // [slot][half][lane]
    const uint16_t *rows = reinterpret_cast<const uint16_t *>(dec_smem + BAR_BYTES + ring_n * HEAD_BYTES);
    const uint32_t rent = rb / 2u;                                                            // entries per slot
    auto tx_bar = [&](int k) { return bars + 8u * k; };                         // row bytes landed
    auto full_bar = [&](int k) { return bars + 8u * (MAX_RING + k); };          // heads written (helper -> decoder)
    auto empty_bar = [&](int k) { return bars + 8u * (2 * MAX_RING + k); };     // slot consumed (decoder -> helper)
    if (threadIdx.x == 0) {
        for (int k = 0; k < ring_n; ++k) {
            mbar_init(tx_bar(k), 1);
            mbar_init(full_bar(k), 32);
            mbar_init(empty_bar(k), 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const l3c_dec_stream_t st = streams[blockIdx.x];
    uint32_t last, upd_end;
    if (!chunk_of(st.n_sym, first, count, last, upd_end)) return;
    const uint32_t n = last - first;
    const uint32_t s = ((uint32_t)L + 255u) / 256u;                             // entries per bucket, <= 128

    if (warp == 1) {
        // ============================ helper warp ============================
        const uint8_t *table = reinterpret_cast<const uint8_t *>(st.table);
        const int64_t pitch_bytes = 2 * st.row_pitch;
        int k_in = 0, k_out = 0;                  // slot of the next row to request / to index
        uint32_t ph_in = 0, ph_out = 0;           // and the parity of that slot's current use
        for (uint32_t q = 0; q < n + (uint32_t)ring_n - 1u; ++q) {
            if (q < n) {
                if (q >= (uint32_t)ring_n) mbar_wait(empty_bar(k_in), ph_in ^ 1u);   // the decoder is done with it
                if (lane == 0)
                    stage_row(smem_u32(rows + (size_t)k_in * rent), table + (int64_t)(first + q) * pitch_bytes, rb,
                              tx_bar(k_in));
                if (++k_in == ring_n) { k_in = 0; ph_in ^= 1u; }
            }
            if (q + 1u >= (uint32_t)ring_n) {     // row q - (ring_n - 1): build its heads
                mbar_wait(tx_bar(k_out), ph_out);
                const uint16_t *row = rows + (size_t)k_out * rent;
                uint32_t h[8];
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const uint32_t j = 8u * lane + jj, m = j * s;
                    h[jj] = (m < (uint32_t)L) ? (((uint32_t)row[m] << 16) | j) : 0u;
                }
                heads[k_out][0][lane] = make_uint4(h[0], h[1], h[2], h[3]);
                heads[k_out][1][lane] = make_uint4(h[4], h[5], h[6], h[7]);
                mbar_arrive(full_bar(k_out));
                if (++k_out == ring_n) { k_out = 0; ph_out ^= 1u; }
            }
        }
        return;
    }

    // ============================ decoder warp ============================
    BitSource src;
    CoderState cs;
    const uint32_t bit0 = open_stream(st, first, src, cs);
    uint16_t *__restrict__ sym_out = reinterpret_cast<uint16_t *>(st.sym_out);
    int k = 0;
    uint32_t ph = 0;
    for (uint32_t i = first; i < last; ++i) {
        mbar_wait(full_bar(k), ph);
        mbar_wait(tx_bar(k), ph);                 // complete already; makes the staged bytes visible to this warp
        // level 1: the bucket
        const uint4 a = heads[k][0][lane], b = heads[k][1][lane];
        const uint32_t hk[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        const uint32_t m0 = (exact_step(hk, cs, src, lane, false) & 0xFFFFu) * s;
        // level 2: the entry inside it
        const uint16_t *row = rows + (size_t)k * rent;
        const uint32_t m_end = min(m0 + s, (uint32_t)L);
        uint32_t pk[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const uint32_t m = m0 + lane + 32u * t;
            pk[t] = 0u;
            if (m < m_end) {
                const uint32_t hi = (m + 1u == (uint32_t)L) ? 0x10000u : (uint32_t)row[m + 1u];
                pk[t] = ((uint32_t)row[m] << 16) | ((hi - 1u) & 0xFFFFu);
            }
        }
        const uint32_t top = exact_step(pk, cs, src, lane, i < upd_end);
        int c = 0;
#pragma unroll
        for (int t = 0; t < 4; ++t) c += (m0 + lane + 32u * t < m_end && pk[t] <= top) ? 1 : 0;
        const int tot = __reduce_add_sync(FULL, c);   // >= 1: entry m0 passes
        mbar_arrive(empty_bar(k));
        if (lane == 0) sym_out[i] = (uint16_t)(m0 + (uint32_t)tot - 1u);
        if (++k == ring_n) { k = 0; ph ^= 1u; }
    }
    if (lane == 0) save_stream(st, cs, src, bit0);
}

}  // namespace wide

// ---------------------------------------------------------------------------------------------
// gather the variable-length code streams into one contiguous blob (container layout, byte offsets)
// ---------------------------------------------------------------------------------------------
constexpr int PACK_CHUNK = 16384;
constexpr int PACK_GRID_X = 64;
// grid = (PACK_GRID_X, streams): every CTA walks its stream in strides of PACK_GRID_X chunks, so a
// stream of ANY length is copied completely (a fixed 256-chunk grid used to stop at 4 MiB)
__global__ void pack_streams_kernel(const l3c_enc_stream_t *__restrict__ streams,
                                    const uint32_t *__restrict__ lens,
                                    const uint64_t *__restrict__ dst_off, uint8_t *__restrict__ blob) {
    const l3c_enc_stream_t st = streams[blockIdx.y];
    const uint32_t len = min(lens[blockIdx.y], st.out_cap);
    uint8_t *dst = blob + dst_off[blockIdx.y];
    for (uint64_t b0 = (uint64_t)blockIdx.x * PACK_CHUNK; b0 < len; b0 += (uint64_t)gridDim.x * PACK_CHUNK) {
        // 64-bit positions: a 32-bit i would wrap past 2^32 - 1 in the last chunk of a slot of almost 4 GiB
        const uint64_t b1 = min(b0 + (uint64_t)PACK_CHUNK, (uint64_t)len);
        for (uint64_t i = b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = st.out[i];
    }
}

// splice of region updates: one warp per chunk of SPLICE_CHUNK bytes of a segment, so a segment of one short stream
// takes one warp and a long run of unchanged streams many.  seg = the n_seg segments [n_seg][4] followed by chunk0
// [n_seg + 1], the first chunk of every segment (a prefix sum; chunk0[n_seg] = all chunks); a segment of src 1 has at
// least one chunk, whose warp also writes its length field.
constexpr int SPLICE_CHUNK = 4096;
constexpr int SPLICE_THREADS = 256;
__global__ void __launch_bounds__(SPLICE_THREADS)
splice_streams_kernel(const int64_t *__restrict__ seg, int n_seg, const uint8_t *__restrict__ old,
                      const uint8_t *__restrict__ slots, uint8_t *__restrict__ out) {
    const int64_t *chunk0 = seg + 4 * (int64_t)n_seg;
    const int64_t total = chunk0[n_seg];
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (SPLICE_THREADS / 32);
    for (int64_t w = (int64_t)blockIdx.x * (SPLICE_THREADS / 32) + (threadIdx.x >> 5); w < total; w += warps) {
        int lo = 0, hi = n_seg - 1;                    // the segment s with chunk0[s] <= w < chunk0[s + 1]
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (chunk0[mid] <= w) lo = mid; else hi = mid - 1;
        }
        const int64_t kind = seg[4 * lo], n = seg[4 * lo + 3];
        const int64_t b0 = (w - chunk0[lo]) * SPLICE_CHUNK, b1 = min(b0 + SPLICE_CHUNK, n);
        const uint8_t *src = (kind ? slots : old) + seg[4 * lo + 1];
        uint8_t *dst = out + seg[4 * lo + 2];
        if (kind && b0 == 0 && lane < 4)                  // the new stream's u32 length, little-endian
            dst[lane - 4] = (uint8_t)((uint64_t)n >> (8 * lane));
        for (int64_t i = b0 + lane; i < b1; i += 32) dst[i] = src[i];
    }
}

// ---- layout and splice of region updates from device-resident lengths (l3c_update_layout, l3c_splice_streams_dev)
constexpr int LAYOUT_THREADS = 256;
constexpr int64_t UPD_SLOT_OVERFLOW = 1, UPD_INCONSISTENT = 2;

// Exclusive scan of (a, b) over the CTA; *ta / *tb get the CTA's totals.  ws: LAYOUT_THREADS / 32 pairs of shared
// memory; every thread calls it.
__device__ __forceinline__ void block_scan2(int64_t a, int64_t b, int64_t *ws, int64_t &ea, int64_t &eb,
                                            int64_t &ta, int64_t &tb) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int NW = LAYOUT_THREADS / 32;
    int64_t x = a, y = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t px = __shfl_up_sync(0xffffffffu, x, o), py = __shfl_up_sync(0xffffffffu, y, o);
        if (lane >= o) x += px, y += py;
    }
    if (lane == 31) ws[2 * wid] = x, ws[2 * wid + 1] = y;
    __syncthreads();
    if (wid == 0) {
        int64_t u = lane < NW ? ws[2 * lane] : 0, v = lane < NW ? ws[2 * lane + 1] : 0;
#pragma unroll
        for (int o = 1; o < NW; o <<= 1) {
            const int64_t pu = __shfl_up_sync(0xffffffffu, u, o), pv = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) u += pu, v += pv;
        }
        if (lane < NW) ws[2 * lane] = u, ws[2 * lane + 1] = v;
    }
    __syncthreads();
    ea = (wid ? ws[2 * wid - 2] : 0) + x - a;
    eb = (wid ? ws[2 * wid - 1] : 0) + y - b;
    ta = ws[2 * NW - 2];
    tb = ws[2 * NW - 1];
    __syncthreads();                                   // ws is reused by the next call
}

// a container's segments [first_seg, first_seg + 2 n_new + 1) lie in the segment array of n_seg
__device__ __forceinline__ bool update_segs_ok(const l3c_update_container_t &c, int64_t n_seg) {
    return c.n_new >= 0 && c.n_new <= n_seg && c.first_seg >= 0 && c.first_seg <= n_seg - (2 * c.n_new + 1);
}

__device__ __forceinline__ bool update_container_ok(const l3c_update_container_t &c, int64_t n_streams, int64_t n_seg) {
    return update_segs_ok(c, n_seg) && c.first_stream >= 0 && c.n_streams >= 0 && c.first_stream <= n_streams - c.n_streams &&
           c.n_new <= c.n_streams && c.old_base >= 0 && c.old_bytes >= 0 && c.out_base >= 0 && c.out_cap >= 0;
}

__global__ void __launch_bounds__(LAYOUT_THREADS)
update_layout_kernel(const l3c_update_container_t *__restrict__ conts, const l3c_update_stream_t *__restrict__ streams,
                     int64_t n_streams, const int32_t *__restrict__ new_len, const int64_t *__restrict__ slot_off,
                     const int64_t *__restrict__ caps, int64_t n_new, int64_t *__restrict__ seg,
                     int64_t *__restrict__ chunk0, int64_t n_seg, int64_t *__restrict__ info, int n_containers) {
    __shared__ int64_t ws[2 * (LAYOUT_THREADS / 32)];
    __shared__ int64_t err;
    const int k = blockIdx.x;
    const l3c_update_container_t c = conts[k];
    if (threadIdx.x == 0) err = 0;
    __syncthreads();
    if (!update_container_ok(c, n_streams, n_seg)) {
        // nothing of this container is placed: no segments, and no chunks where its chunk total can be located
        if (threadIdx.x == 0) {
            info[k] = 0;
            if (update_segs_ok(c, n_seg)) chunk0[c.first_seg + k + 2 * c.n_new + 1] = 0;
            atomicOr((unsigned long long *)(info + n_containers), (unsigned long long)UPD_INCONSISTENT);
        }
        return;
    }
    int64_t *sg = seg + 4 * c.first_seg;
    const int64_t m = c.n_new, ns = 2 * m + 1;
    // ---- new offsets: one chunk of LAYOUT_THREADS streams per step, the running sums carried across
    int64_t base_len = 0, base_new = 0;
    for (int64_t s0 = 0; s0 < c.n_streams; s0 += LAYOUT_THREADS) {
        const int64_t s = s0 + threadIdx.x;
        int64_t len = 0, is_new = 0;
        l3c_update_stream_t st{};
        if (s < c.n_streams) {
            st = streams[c.first_stream + s];
            len = st.old_len;
            if (st.src >= 0) {
                is_new = 1;
                if (st.src >= n_new) {
                    atomicOr((unsigned long long *)&err, (unsigned long long)UPD_INCONSISTENT);
                    len = 0;
                } else {
                    len = new_len[st.src];
                    if (len < 0 || len > caps[st.src]) atomicOr((unsigned long long *)&err, (unsigned long long)UPD_SLOT_OVERFLOW);
                }
            }
        }
        int64_t ex_len, ex_new, t_len, t_new;
        block_scan2(len, is_new, ws, ex_len, ex_new, t_len, t_new);
        const int64_t j = base_new + ex_new;
        if (is_new && j < m && st.src < n_new) {
            const int64_t off = c.out_base + st.fixed_off + base_len + ex_len;
            int64_t *a = sg + 4 * (2 * j + 1), *b = a + 4;
            a[0] = 1, a[1] = slot_off[st.src], a[2] = off, a[3] = len;
            b[0] = 0, b[1] = c.old_base + st.old_off + st.old_len, b[2] = off + len;       // b[3] below
        }
        base_len += t_len;
        base_new += t_new;
    }
    const int64_t total = c.fixed_total + base_len;
    if (threadIdx.x == 0) {
        sg[0] = 0, sg[1] = c.old_base, sg[2] = c.out_base;
        if (base_new != m || total > c.out_cap) atomicOr((unsigned long long *)&err, (unsigned long long)UPD_INCONSISTENT);
        info[k] = total;
    }
    __syncthreads();
    // ---- every run ends at the length field of the next new stream or at the container's end: unchanged bytes
    // keep their distances, so its size follows from the destinations
    if (base_new == m)
        for (int64_t j = threadIdx.x; j <= m; j += LAYOUT_THREADS) {
            const int64_t end = j < m ? sg[4 * (2 * j + 1) + 2] - 4 : c.out_base + total;
            sg[4 * (2 * j) + 3] = end - sg[4 * (2 * j) + 2];
            if (end < sg[4 * (2 * j) + 2]) atomicOr((unsigned long long *)&err, (unsigned long long)UPD_INCONSISTENT);
        }
    __syncthreads();
    const bool bad = err != 0;
    // ---- chunks per segment (SPLICE_CHUNK bytes each, one for an empty new stream: its length field), prefix
    int64_t *ch = chunk0 + c.first_seg + k;
    int64_t base = 0;
    for (int64_t i0 = 0; i0 < ns; i0 += LAYOUT_THREADS) {
        const int64_t i = i0 + threadIdx.x;
        int64_t n = 0;
        if (i < ns && !bad) {
            const int64_t b = sg[4 * i + 3];
            n = b > 0 ? (b + SPLICE_CHUNK - 1) / SPLICE_CHUNK : sg[4 * i];
        }
        int64_t ex, unused, t, t2;
        block_scan2(n, 0, ws, ex, unused, t, t2);
        if (i < ns) ch[i] = base + ex;
        base += t;
    }
    if (threadIdx.x == 0) {
        ch[ns] = base;
        if (bad) atomicOr((unsigned long long *)(info + n_containers), (unsigned long long)err);
    }
}

__global__ void __launch_bounds__(SPLICE_THREADS)
splice_streams_dev_kernel(const l3c_update_container_t *__restrict__ conts, int k0, const int64_t *__restrict__ seg,
                          const int64_t *__restrict__ chunk0, int64_t n_seg, const uint8_t *__restrict__ old,
                          int64_t old_bytes, const uint8_t *__restrict__ slots, int64_t slot_bytes,
                          uint8_t *__restrict__ out, int64_t out_bytes, int64_t *__restrict__ flag) {
    const int k = k0 + blockIdx.y;
    const l3c_update_container_t c = conts[k];
    if (!update_segs_ok(c, n_seg)) return;            // l3c_update_layout flagged it
    const int64_t ns = 2 * c.n_new + 1;
    const int64_t *sg = seg + 4 * c.first_seg, *ch = chunk0 + c.first_seg + k;
    const int64_t total = ch[ns];
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (SPLICE_THREADS / 32);
    for (int64_t w = (int64_t)blockIdx.x * (SPLICE_THREADS / 32) + (threadIdx.x >> 5); w < total; w += warps) {
        int64_t lo = 0, hi = ns - 1;                   // the segment s with ch[s] <= w < ch[s + 1]
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) >> 1;
            if (ch[mid] <= w) lo = mid; else hi = mid - 1;
        }
        const int64_t kind = sg[4 * lo], so = sg[4 * lo + 1], d = sg[4 * lo + 2], n = sg[4 * lo + 3];
        const int64_t s_lo = kind ? 0 : c.old_base, s_hi = kind ? slot_bytes : min(c.old_base + c.old_bytes, old_bytes);
        const int64_t d_lo = max(c.out_base, (int64_t)0), d_hi = min(c.out_base + c.out_cap, out_bytes);
        const bool ok = (kind == 0 || kind == 1) && n >= 0 && (kind == 0 || n <= 0xffffffffll) && so >= s_lo &&
                        so <= s_hi - n && d - 4 * kind >= d_lo && d <= d_hi - n;
        if (!ok) {
            if (lane == 0) atomicOr((unsigned long long *)flag, (unsigned long long)UPD_INCONSISTENT);
            continue;
        }
        const int64_t b0 = (w - ch[lo]) * SPLICE_CHUNK, b1 = min(b0 + SPLICE_CHUNK, n);
        const uint8_t *src = (kind ? slots : old) + so;
        uint8_t *dst = out + d;
        if (kind && b0 == 0 && lane < 4)                  // the new stream's u32 length, little-endian
            dst[lane - 4] = (uint8_t)((uint64_t)n >> (8 * lane));
        for (int64_t i = b0 + lane; i < b1; i += 32) dst[i] = src[i];
    }
}

// intervals from a shared 256-entry LUT (uniform prior: every pixel has the same CDF row)
__global__ void lut_intervals_kernel(const uint8_t *__restrict__ sym, const uint32_t *__restrict__ lut,
                                     int64_t n, uint32_t *__restrict__ iv) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) iv[i] = __ldg(lut + sym[i]);
}

}  // namespace l3c

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
namespace l3c {
// streams per CTA of the helper-warp decoders and of the encoder: a test knob, else an environment variable (read
// once), else the default
static int spc_from_env(const char *name, int dflt) {
    const char *e = getenv(name);
    const int v = e ? atoi(e) : dflt;
    return (v == 1 || v == 2 || v == 4) ? v : dflt;
}

std::atomic<int> g_enc_spc{0};   // l3c_set_encoder_streams_per_cta: 0 = L3C_ENC_SPC / the default
// 4 streams per CTA: at the 288 streams of a bench batch the fastest in isolation, and in the pipelined step ~5 %
// faster than 1 (DESIGN §7)
constexpr int DEFAULT_ENC_SPC = 4;
static int encoder_spc() {
    static const int env_spc = spc_from_env("L3C_ENC_SPC", DEFAULT_ENC_SPC);
    const int forced = g_enc_spc.load(std::memory_order_relaxed);
    return forced ? forced : env_spc;
}
}  // namespace l3c

extern "C" int l3c_ac_encode_streams(const l3c_enc_stream_t *streams_dev, int n_streams,
                                     uint32_t *out_len_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_encode_streams: n_streams=%d", n_streams);
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && out_len_dev, "l3c_ac_encode_streams: null pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    const int spc = encoder_spc();
    if (spc == 4)
        ac_encode_kernel<4><<<ceil_div(n_streams, 4), 256, 0, st>>>(streams_dev, n_streams, out_len_dev);
    else if (spc == 2)
        ac_encode_kernel<2><<<ceil_div(n_streams, 2), 128, 0, st>>>(streams_dev, n_streams, out_len_dev);
    else
        ac_encode_kernel<1><<<n_streams, 64, 0, st>>>(streams_dev, n_streams, out_len_dev);
    L3C_LAUNCH_CHECK("ac_encode_kernel");
    return L3C_OK;
}

extern "C" int l3c_ac_encode_streams_seek(const l3c_enc_stream_t *streams_dev, int n_streams, uint32_t *out_len_dev,
                                          uint32_t every, uint32_t *const *points_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_encode_streams_seek: n_streams=%d", n_streams);
    L3C_REQUIRE(every >= 32u && every % 32u == 0u, "l3c_ac_encode_streams_seek: every=%u is not a positive multiple "
                "of 32", every);
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && out_len_dev && points_dev, "l3c_ac_encode_streams_seek: null pointer");
    const cudaStream_t st = (cudaStream_t)stream;
    const int spc = encoder_spc();
    if (spc == 4)
        ac_encode_seek_kernel<4><<<ceil_div(n_streams, 4), 256, 0, st>>>(streams_dev, n_streams, out_len_dev, every,
                                                                          points_dev);
    else if (spc == 2)
        ac_encode_seek_kernel<2><<<ceil_div(n_streams, 2), 128, 0, st>>>(streams_dev, n_streams, out_len_dev, every,
                                                                          points_dev);
    else
        ac_encode_seek_kernel<1><<<n_streams, 64, 0, st>>>(streams_dev, n_streams, out_len_dev, every, points_dev);
    L3C_LAUNCH_CHECK("ac_encode_seek_kernel");
    return L3C_OK;
}

extern "C" int l3c_set_encoder_streams_per_cta(int spc) {
    L3C_REQUIRE(spc == 0 || spc == 1 || spc == 2 || spc == 4,
                "l3c_set_encoder_streams_per_cta: spc=%d not in {0, 1, 2, 4}", spc);
    l3c::g_enc_spc.store(spc);
    return L3C_OK;
}

namespace l3c {
std::atomic<int> g_dec_spc{0};   // l3c_set_decoder_streams_per_cta: 0 = L3C_DEC_SPC / the default

// streams per CTA of the helper-warp decoders: the knob, else L3C_DEC_SPC (read once), else 2.  A CTA of 2 streams
// holds the decoder warps 0-1 and their helpers 2-3.  In the pipelined step, where the decoders of four batches share
// their SM group at 16 warps per SM, that decodes ~6 % faster than one stream per CTA, and 4 streams no better than 2
// (DESIGN §7).
constexpr int DEFAULT_DEC_SPC = 2;
static int decoder_spc() {
    static const int env_spc = spc_from_env("L3C_DEC_SPC", DEFAULT_DEC_SPC);
    const int forced = g_dec_spc.load(std::memory_order_relaxed);
    return forced ? forced : env_spc;
}

template <bool FULLROW, bool SEG = false>
void launch_decode(const l3c_dec_stream_t *streams, int n, int L, uint32_t first, uint32_t count, int spc,
                   cudaStream_t st) {
    using v3::ac_decode_kernel;
    using v3::STREAM_SMEM;
    if (spc == 4)
        ac_decode_kernel<FULLROW, 4, SEG><<<ceil_div(n, 4), 256, 4 * STREAM_SMEM, st>>>(streams, n, L, first, count);
    else if (spc == 2)
        ac_decode_kernel<FULLROW, 2, SEG><<<ceil_div(n, 2), 128, 2 * STREAM_SMEM, st>>>(streams, n, L, first, count);
    else
        ac_decode_kernel<FULLROW, 1, SEG><<<n, 64, STREAM_SMEM, st>>>(streams, n, L, first, count);
}
}  // namespace l3c

extern "C" int l3c_set_decoder_streams_per_cta(int spc) {
    L3C_REQUIRE(spc == 0 || spc == 1 || spc == 2 || spc == 4,
                "l3c_set_decoder_streams_per_cta: spc=%d not in {0, 1, 2, 4}", spc);
    l3c::g_dec_spc.store(spc);
    return L3C_OK;
}

namespace l3c {
// L > 256: the descriptors are checked on the host first (row pitch, alignment of the rows and of the uint16
// output), so a bad one is L3C_EINVAL instead of a misaligned bulk copy; this waits for `st`.
static int decode_wide(const l3c_dec_stream_t *streams_dev, int n, int L, uint32_t first, uint32_t count,
                       cudaStream_t st) {
    using wide::ac_decode_wide_kernel;
    std::vector<l3c_dec_stream_t> d((size_t)n);
    L3C_CUDA(cudaMemcpyAsync(d.data(), streams_dev, sizeof(l3c_dec_stream_t) * (size_t)n, cudaMemcpyDeviceToHost, st));
    L3C_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) {
        const int64_t p = d[(size_t)i].row_pitch;
        L3C_REQUIRE(p == 0 || (p % 8 == 0 && p >= L),
                    "l3c_ac_decode_streams: stream %d: row_pitch=%lld for L=%d (L > 256 needs 0 or a multiple of 8 "
                    ">= L)", i, (long long)p, L);
        L3C_REQUIRE((reinterpret_cast<uintptr_t>(d[(size_t)i].table) & 15u) == 0 &&
                        (reinterpret_cast<uintptr_t>(d[(size_t)i].sym_out) & 1u) == 0,
                    "l3c_ac_decode_streams: stream %d: table must be 16-byte and sym_out 2-byte aligned for L > 256", i);
    }
    static int optin_dev[64] = {};
    int &optin = optin_dev[current_device_slot()];
    if (!optin) {   // opt in once per device to all the shared memory a block may have
        int dev = 0, v = 0;
        L3C_CUDA(cudaGetDevice(&dev));
        L3C_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        L3C_CUDA(cudaFuncSetAttribute(ac_decode_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
        optin = v;
    }
    // as many row slots as fit, 2 to MAX_RING (3 at L = 32768 with 227 KB)
    const int ring_n = (int)std::min<size_t>(wide::MAX_RING, ((size_t)optin - wide::BAR_BYTES) /
                                                                 (wide::HEAD_BYTES + wide::row_bytes(L)));
    L3C_REQUIRE(ring_n >= 2, "l3c_ac_decode_streams: L=%d needs %zu bytes of shared memory, the device offers %d", L,
                wide::smem_bytes(2, L), optin);
    ac_decode_wide_kernel<<<n, 64, wide::smem_bytes(ring_n, L), st>>>(streams_dev, L, ring_n, first, count);
    L3C_LAUNCH_CHECK("ac_decode_wide_kernel");
    return L3C_OK;
}
}  // namespace l3c

extern "C" int l3c_ac_decode_streams(const l3c_dec_stream_t *streams_dev, int n_streams, int L,
                                     uint32_t first, uint32_t count, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_decode_streams: n_streams=%d", n_streams);
    L3C_REQUIRE(L >= 1 && L <= 32768, "l3c_ac_decode_streams: L=%d not in [1,32768]", L);
    if (n_streams == 0 || count == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev, "l3c_ac_decode_streams: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (L > 256) return decode_wide(streams_dev, n_streams, L, first, count, st);
    if (L <= 32) {
        ac_decode32_kernel<<<n_streams, 32, 0, st>>>(streams_dev, n_streams, L, first, count);
    } else {
        const int spc = decoder_spc();
        static bool configured_dev[64] = {};
        bool &configured = configured_dev[current_device_slot()];
        if (!configured) {   // the SPC = 4 variants are the ones above 48 KB of shared memory
            L3C_CUDA(cudaFuncSetAttribute(v3::ac_decode_kernel<true, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          4 * v3::STREAM_SMEM));
            L3C_CUDA(cudaFuncSetAttribute(v3::ac_decode_kernel<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          4 * v3::STREAM_SMEM));
            configured = true;
        }
        if (L == 256)
            launch_decode<true>(streams_dev, n_streams, L, first, count, spc, st);
        else
            launch_decode<false>(streams_dev, n_streams, L, first, count, spc, st);
    }
    L3C_LAUNCH_CHECK("ac_decode_kernel");
    return L3C_OK;
}

extern "C" int l3c_ac_decode_streams_coarse(const l3c_dec_stream_t *streams_dev, int n_streams,
                                            const float *targets_dev, uint32_t first, uint32_t count, void *stream) {
    using namespace l3c;
    using coarse::ac_decode_coarse_kernel;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_decode_streams_coarse: n_streams=%d", n_streams);
    if (n_streams == 0 || count == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && targets_dev, "l3c_ac_decode_streams_coarse: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int spc = decoder_spc();
    if (spc == 4)
        ac_decode_coarse_kernel<4><<<ceil_div(n_streams, 4), 256, coarse::smem_bytes(4), st>>>(streams_dev, n_streams,
                                                                                           targets_dev, first, count);
    else if (spc == 2)
        ac_decode_coarse_kernel<2><<<ceil_div(n_streams, 2), 128, coarse::smem_bytes(2), st>>>(streams_dev, n_streams,
                                                                                           targets_dev, first, count);
    else
        ac_decode_coarse_kernel<1><<<n_streams, 64, coarse::smem_bytes(1), st>>>(streams_dev, n_streams, targets_dev,
                                                                                 first, count);
    // logged under the decoder family's name, like every v3 variant: a decode makes the same launches whether its
    // RGB scale reads coarse records or full rows
    L3C_LAUNCH_CHECK("ac_decode_kernel");
    return L3C_OK;
}

// segment mode: every descriptor is decoded whole (first 0, every symbol), from its seek point when `state` is set
extern "C" int l3c_ac_decode_segments(const l3c_dec_stream_t *segs_dev, int n_segs, int L, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_segs >= 0, "l3c_ac_decode_segments: n_segs=%d", n_segs);
    L3C_REQUIRE(L >= 1 && L <= 256, "l3c_ac_decode_segments: L=%d not in [1,256]", L);
    if (n_segs == 0) return L3C_OK;
    L3C_REQUIRE(segs_dev, "l3c_ac_decode_segments: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (L <= 32) {
        ac_decode32_kernel<true><<<n_segs, 32, 0, st>>>(segs_dev, n_segs, L, 0u, 0xFFFFFFFFu);
    } else {
        const int spc = decoder_spc();
        static bool configured_dev[64] = {};
        bool &configured = configured_dev[current_device_slot()];
        if (!configured) {
            L3C_CUDA(cudaFuncSetAttribute(v3::ac_decode_kernel<true, 4, true>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * v3::STREAM_SMEM));
            L3C_CUDA(cudaFuncSetAttribute(v3::ac_decode_kernel<false, 4, true>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * v3::STREAM_SMEM));
            configured = true;
        }
        if (L == 256)
            launch_decode<true, true>(segs_dev, n_segs, L, 0u, 0xFFFFFFFFu, spc, st);
        else
            launch_decode<false, true>(segs_dev, n_segs, L, 0u, 0xFFFFFFFFu, spc, st);
    }
    L3C_LAUNCH_CHECK("ac_decode_segments");
    return L3C_OK;
}

extern "C" int l3c_ac_decode_segments_coarse(const l3c_dec_stream_t *segs_dev, int n_segs, const float *targets_dev,
                                             void *stream) {
    using namespace l3c;
    using coarse::ac_decode_coarse_kernel;
    L3C_REQUIRE(n_segs >= 0, "l3c_ac_decode_segments_coarse: n_segs=%d", n_segs);
    if (n_segs == 0) return L3C_OK;
    L3C_REQUIRE(segs_dev && targets_dev, "l3c_ac_decode_segments_coarse: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int spc = decoder_spc();
    if (spc == 4)
        ac_decode_coarse_kernel<4, true><<<ceil_div(n_segs, 4), 256, coarse::smem_bytes(4), st>>>(
            segs_dev, n_segs, targets_dev, 0u, 0xFFFFFFFFu);
    else if (spc == 2)
        ac_decode_coarse_kernel<2, true><<<ceil_div(n_segs, 2), 128, coarse::smem_bytes(2), st>>>(
            segs_dev, n_segs, targets_dev, 0u, 0xFFFFFFFFu);
    else
        ac_decode_coarse_kernel<1, true><<<n_segs, 64, coarse::smem_bytes(1), st>>>(segs_dev, n_segs, targets_dev, 0u,
                                                                                    0xFFFFFFFFu);
    L3C_LAUNCH_CHECK("ac_decode_segments_coarse");
    return L3C_OK;
}

extern "C" int l3c_pack_streams(const l3c_enc_stream_t *streams_dev, const uint32_t *len_dev,
                                const uint64_t *dst_off_dev, int n_streams, uint8_t *blob_dev,
                                void *stream) {
    using namespace l3c;
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && len_dev && dst_off_dev && blob_dev && n_streams > 0, "l3c_pack_streams: bad arguments");
    // one stream per grid row: a container of more streams than grid.y holds (a large tiled image) takes several
    // launches of at most 65535 streams each
    for (int first = 0; first < n_streams; first += 65535) {
        dim3 grid(PACK_GRID_X, n_streams - first < 65535 ? n_streams - first : 65535);
        pack_streams_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(streams_dev + first, len_dev + first,
                                                                     dst_off_dev + first, blob_dev);
        L3C_LAUNCH_CHECK("pack_streams_kernel");
    }
    return L3C_OK;
}

extern "C" int l3c_splice_streams(const uint8_t *old_dev, int64_t old_bytes, const uint8_t *slots_dev,
                                  int64_t slot_bytes, const int64_t *seg_host, int64_t *seg_dev, int n_seg,
                                  uint8_t *out_dev, int64_t out_bytes, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_seg >= 0, "l3c_splice_streams: %d segments", n_seg);
    if (n_seg == 0) return L3C_OK;
    L3C_REQUIRE(old_dev && slots_dev && seg_host && seg_dev && out_dev, "l3c_splice_streams: null pointer");
    L3C_REQUIRE(((uintptr_t)seg_dev & 7) == 0, "l3c_splice_streams: seg_dev must be 8-byte aligned");
    // every destination, a new stream's length field included, as [begin, end) for the overlap check
    std::vector<std::pair<int64_t, int64_t>> dst(n_seg);
    for (int s = 0; s < n_seg; ++s) {
        const int64_t kind = seg_host[4 * s], so = seg_host[4 * s + 1], d = seg_host[4 * s + 2], n = seg_host[4 * s + 3];
        const int64_t src_bytes = kind ? slot_bytes : old_bytes;
        L3C_REQUIRE(kind == 0 || kind == 1, "l3c_splice_streams: segment %d has source %lld", s, (long long)kind);
        L3C_REQUIRE(n >= 0 && (kind == 0 || n <= 0xffffffffll), "l3c_splice_streams: segment %d of %lld bytes", s,
                    (long long)n);
        L3C_REQUIRE(so >= 0 && so <= src_bytes - n, "l3c_splice_streams: segment %d reads [%lld, %lld) of a %lld-byte "
                    "source", s, (long long)so, (long long)(so + n), (long long)src_bytes);
        L3C_REQUIRE(d - 4 * kind >= 0 && d <= out_bytes - n, "l3c_splice_streams: segment %d writes [%lld, %lld) of a "
                    "%lld-byte output", s, (long long)(d - 4 * kind), (long long)(d + n), (long long)out_bytes);
        dst[s] = {d - 4 * kind, d + n};
    }
    // chunks of every segment, appended to the segments for the kernel
    std::vector<int64_t> buf(seg_host, seg_host + 4 * (size_t)n_seg);
    buf.resize(5 * (size_t)n_seg + 1);
    int64_t chunks = 0;
    for (int s = 0; s < n_seg; ++s) {
        buf[4 * (size_t)n_seg + s] = chunks;
        const int64_t n = seg_host[4 * s + 3];
        chunks += n > 0 ? (n + SPLICE_CHUNK - 1) / SPLICE_CHUNK : seg_host[4 * s];
    }
    buf[5 * (size_t)n_seg] = chunks;
    std::sort(dst.begin(), dst.end());
    for (int s = 1; s < n_seg; ++s)
        L3C_REQUIRE(dst[s].first >= dst[s - 1].second, "l3c_splice_streams: destinations [%lld, %lld) and [%lld, %lld) "
                    "overlap", (long long)dst[s - 1].first, (long long)dst[s - 1].second, (long long)dst[s].first,
                    (long long)dst[s].second);
    cudaStream_t st = (cudaStream_t)stream;
    if (chunks == 0) return L3C_OK;                        // every segment empty
    // from pageable memory: returns once buf has been read, so it may be freed
    L3C_REQUIRE(cudaMemcpyAsync(seg_dev, buf.data(), buf.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st) ==
                    cudaSuccess, "l3c_splice_streams: segment upload failed");
    const int64_t blocks = (chunks + SPLICE_THREADS / 32 - 1) / (SPLICE_THREADS / 32);
    splice_streams_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), SPLICE_THREADS, 0, st>>>(seg_dev, n_seg,
                                                                                                old_dev, slots_dev,
                                                                                                out_dev);
    L3C_LAUNCH_CHECK("splice_streams_kernel");
    return L3C_OK;
}

extern "C" int l3c_update_layout(const l3c_update_container_t *conts_dev, int n_containers,
                                 const l3c_update_stream_t *streams_dev, int64_t n_streams, const int32_t *new_len_dev,
                                 const int64_t *slot_off_dev, const int64_t *caps_dev, int64_t n_new, int64_t *seg_dev,
                                 int64_t *chunk0_dev, int64_t n_seg, int64_t *info_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_containers >= 0 && n_streams >= 0 && n_new >= 0 && n_seg >= 0,
                "l3c_update_layout: n_containers=%d n_streams=%lld n_new=%lld n_seg=%lld", n_containers,
                (long long)n_streams, (long long)n_new, (long long)n_seg);
    L3C_REQUIRE(info_dev, "l3c_update_layout: null info_dev");
    L3C_REQUIRE(n_containers == 0 || (conts_dev && streams_dev && seg_dev && chunk0_dev &&
                                      (n_new == 0 || (new_len_dev && slot_off_dev && caps_dev))),
                "l3c_update_layout: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    L3C_CUDA(cudaMemsetAsync(info_dev + n_containers, 0, sizeof(int64_t), st));
    if (n_containers == 0) return L3C_OK;
    update_layout_kernel<<<n_containers, LAYOUT_THREADS, 0, st>>>(conts_dev, streams_dev, n_streams, new_len_dev,
                                                                   slot_off_dev, caps_dev, n_new, seg_dev, chunk0_dev,
                                                                   n_seg, info_dev, n_containers);
    L3C_LAUNCH_CHECK("update_layout_kernel");
    return L3C_OK;
}

extern "C" int l3c_splice_streams_dev(const l3c_update_container_t *conts_dev, int n_containers,
                                      const int64_t *seg_dev, const int64_t *chunk0_dev, int64_t n_seg,
                                      const uint8_t *old_dev, int64_t old_bytes, const uint8_t *slots_dev, int64_t slot_bytes, uint8_t *out_dev,
                                      int64_t out_bytes, int64_t max_chunks, int64_t *flag_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_containers >= 0 && n_seg >= 0 && old_bytes >= 0 && slot_bytes >= 0 && out_bytes >= 0 &&
                    max_chunks >= 0,
                "l3c_splice_streams_dev: n_containers=%d n_seg=%lld old_bytes=%lld slot_bytes=%lld out_bytes=%lld "
                "max_chunks=%lld", n_containers, (long long)n_seg, (long long)old_bytes, (long long)slot_bytes,
                (long long)out_bytes, (long long)max_chunks);
    if (n_containers == 0 || max_chunks == 0) return L3C_OK;
    L3C_REQUIRE(conts_dev && seg_dev && chunk0_dev && old_dev && slots_dev && out_dev && flag_dev,
                "l3c_splice_streams_dev: null pointer");
    const int64_t blocks = (max_chunks + SPLICE_THREADS / 32 - 1) / (SPLICE_THREADS / 32);
    for (int k0 = 0; k0 < n_containers; k0 += 65535) {
        dim3 grid((unsigned)(blocks < 65535 ? blocks : 65535), n_containers - k0 < 65535 ? n_containers - k0 : 65535);
        splice_streams_dev_kernel<<<grid, SPLICE_THREADS, 0, (cudaStream_t)stream>>>(
            conts_dev, k0, seg_dev, chunk0_dev, n_seg, old_dev, old_bytes, slots_dev, slot_bytes, out_dev, out_bytes,
            flag_dev);
        L3C_LAUNCH_CHECK("splice_streams_dev_kernel");
    }
    return L3C_OK;
}

extern "C" int l3c_lut_intervals(const uint8_t *sym_dev, const uint32_t *lut_dev, int64_t n,
                                 uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(sym_dev && lut_dev && intervals_dev && (const void *)sym_dev != (const void *)intervals_dev &&
                    (const void *)lut_dev != (const void *)intervals_dev && fits_grid_x(n),
                "l3c_lut_intervals: bad arguments (n=%lld)", (long long)n);
    if (n == 0) return L3C_OK;
    lut_intervals_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(sym_dev, lut_dev, n,
                                                                                       intervals_dev);
    L3C_LAUNCH_CHECK("lut_intervals_kernel");
    return L3C_OK;
}
