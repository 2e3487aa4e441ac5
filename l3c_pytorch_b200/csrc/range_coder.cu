// range_coder.cu -- batched binary arithmetic coder for sm_90a: one warp per stream.
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
//   * the encoder keeps bit emission off its serial chain: per symbol only (low, k, u) is recorded,
//     every 32 symbols the warp packs the 32 bit strings in parallel (one packed scan);
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

#include <atomic>

#include "common.cuh"

namespace l3c {

constexpr unsigned FULL = 0xFFFFFFFFu;
constexpr int ENC_WARPS_PER_CTA = 1;
constexpr int DEC_WARPS_PER_CTA = 1;

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

// Emission is kept OFF the coder's serial dependency chain: the coding loop only records, per symbol,
// the pre-shift `low` and the two shift counts (k decided bits, u underflow shifts) in lane j's
// registers; every 32 symbols the warp turns the 32 records into bits IN PARALLEL:
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

__global__ void __launch_bounds__(32 * ENC_WARPS_PER_CTA)
ac_encode_kernel(const l3c_enc_stream_t *__restrict__ streams, int n_streams,
                 uint32_t *__restrict__ out_len) {
    __shared__ uint32_t s_stage[ENC_WARPS_PER_CTA][STAGE_WORDS];
    const int sid = blockIdx.x * ENC_WARPS_PER_CTA + (threadIdx.x >> 5);
    if (sid >= n_streams) return;
    const int lane = threadIdx.x & 31;
    const l3c_enc_stream_t st = streams[sid];
    const uint32_t *__restrict__ iv = st.intervals;
    const uint32_t n = st.n_sym;

    Emitter em;
    em.stage = s_stage[threadIdx.x >> 5];
    em.pending = 0u;
    em.sink.out = reinterpret_cast<uint32_t *>(st.out);
    em.sink.cap_words = st.out_cap >> 2;
    em.sink.wpos = 0;
    em.sink.acc = 0;
    em.sink.nacc = 0;
    em.sink.lane = lane;

    // Coder state is (low, r = high - low): `high` itself is never needed.  Every renormalisation
    // shift -- "equal MSB" (low <<= 1, high = high << 1 | 1) or "underflow" (the same with the MSBs
    // forced to 0 / 1) -- maps r to 2r + 1 (mod 2^32) and leaves bit 31 of low clear, so
    //     r' = (width << s) - 1,   low' = (low << s) & 0x7FFFFFFF      with width = r + 1, s = k + u.
    uint32_t low = 0u, r = 0xFFFFFFFFu;

    // one coding step (torchac.cpp:171-206); lane j keeps the record of symbol j of the batch
#define L3C_ENC_STEP(j)                                                                            \
    {                                                                                              \
        const uint32_t v = __shfl_sync(FULL, mine, (j));                                           \
        const uint32_t c_lo = v & 0xFFFFu;                                                         \
        const uint32_t c_hi = (v >> 16) + 1u;                                                      \
        /* span * c == r * c + c  (span may be 2^32, keep it out of 32-bit registers) */           \
        const uint32_t hi16 = (uint32_t)(((uint64_t)r * c_hi + c_hi) >> 16);                       \
        const uint32_t lo16 = (uint32_t)(((uint64_t)r * c_lo + c_lo) >> 16);                       \
        const uint32_t width = hi16 - lo16;                /* new high - new low + 1 */            \
        low += lo16;                                                                               \
        const uint32_t high = low + width - 1u;                                                    \
        /* renormalisation: k "equal MSB" shifts, then u "underflow" shifts */                     \
        const uint32_t k = (uint32_t)__clz((int)(low ^ high));                                     \
        const uint32_t u = clz_nz(~shl_c(shl_c(low & ~high, k), 1u));                              \
        if (lane == (j)) {                                                                         \
            rec_low = low;                                                                         \
            rec_ku = k | (u << 8);                                                                 \
        }                                                                                          \
        low = shl_c(shl_c(low, k), u) & 0x7FFFFFFFu;                                               \
        r = shl_c(shl_c(width, k), u) - 1u;                                                        \
    }

    uint32_t next = (lane < n) ? __ldg(iv + lane) : 0u;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t mine = next;
        const uint32_t nb = base + 32 + lane;
        next = (nb < n) ? __ldg(iv + nb) : 0u;              // prefetch the next 32 intervals
        uint32_t rec_low = 0u, rec_ku = 0u;
        if (n - base >= 32u) {
#pragma unroll
            for (int j = 0; j < 32; ++j) L3C_ENC_STEP(j)
        } else {
            const int cnt = (int)(n - base);
#pragma unroll 1
            for (int j = 0; j < cnt; ++j) L3C_ENC_STEP(j)
        }
        em.emit(rec_low, rec_ku & 0xFFu, rec_ku >> 8);
    }
#undef L3C_ENC_STEP

    // termination (torchac.cpp:209-219): one more bit + the owed underflow bits, zero-padded --
    // i.e. a one-bit record met with pending + 1 owed bits
    const uint32_t fin = (low < 0x40000000u) ? 0u : 1u;
    em.pending += 1u;
    em.emit(lane == 0 ? (fin << 31) : 0u, lane == 0 ? 1u : 0u, 0u);
    BitSink &sink = em.sink;
    const uint32_t total = sink.wpos * 4u + (uint32_t)((sink.nacc + 7) >> 3);
    if (sink.nacc > 0) {
        const uint32_t w = (uint32_t)(sink.acc << (32 - sink.nacc));
        if (lane == 0 && sink.wpos < sink.cap_words) sink.out[sink.wpos] = __byte_perm(w, 0, 0x0123);
    }
    if (lane == 0) out_len[sid] = total;
}

// ---------------------------------------------------------------------------------------------
// decoder
// ---------------------------------------------------------------------------------------------

// MSB-first bit reader over a byte stream that may start at ANY address (streams are decoded in
// place from the container): words are fetched from the 4-byte aligned address below the stream and
// the first `8*mis` bits are simply skipped; bytes past the end read as zero (torchac.cpp:109-112).
struct BitSource {
    const uint32_t *base;
    uint32_t end_byte;     // mis + in_len: first byte (relative to base) that is past the stream
    uint32_t wbase;        // word index of the upper half of `win`
    uint64_t win;          // words wbase, wbase+1
    uint32_t nextw;        // word wbase+2, ready to use
    uint32_t raw;          // word wbase+3 as loaded (little-endian, unmasked): consumed one refill
                           // later, so its load latency never lands on the coder's serial chain
    uint32_t pos;          // next unread bit, relative to base; invariant 0 <= pos - 32*wbase < 32

    __device__ __forceinline__ uint32_t load_raw(uint32_t i) const {
        return ((int)end_byte - (int)(4u * i) > 0) ? __ldg(base + i) : 0u;
    }
    __device__ __forceinline__ uint32_t finish(uint32_t w_raw, uint32_t i) const {   // big-endian, zero past the end
        const int rem = (int)end_byte - (int)(4u * i);
        uint32_t w = __byte_perm(w_raw, 0, 0x0123);
        if (rem < 4) w = (rem <= 0) ? 0u : (w & (0xFFFFFFFFu << (8 * (4 - rem))));
        return w;
    }
    __device__ __forceinline__ uint32_t word(uint32_t i) const { return finish(load_raw(i), i); }
    __device__ __forceinline__ uint32_t open(const uint8_t *in, uint32_t len) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(in);
        const uint32_t mis = (uint32_t)(a & 3u);
        base = reinterpret_cast<const uint32_t *>(a - mis);
        end_byte = mis + len;
        return 8u * mis;                                   // bit position of the first code bit
    }
    __device__ __forceinline__ void seek(uint32_t p) {
        wbase = p >> 5;
        win = ((uint64_t)word(wbase) << 32) | (uint64_t)word(wbase + 1);
        nextw = word(wbase + 2);
        raw = load_raw(wbase + 3);
        pos = p;
    }
    // the next 32 bits (not consumed)
    __device__ __forceinline__ uint32_t peek32() const { return (uint32_t)((win << (pos & 31u)) >> 32); }
    __device__ __forceinline__ void skip(uint32_t n) {     // n <= 32
        pos += n;
        if ((pos >> 5) != wbase) {
            win = (win << 32) | (uint64_t)nextw;
            wbase++;
            nextw = finish(raw, wbase + 2);
            raw = load_raw(wbase + 3);
        }
    }
    // same as skip(), written so that it compiles to predicated straight-line code (fast decode loops)
    __device__ __forceinline__ void skip_flat(uint32_t n) {
        pos += n;
        const bool cross = (pos >> 5) != wbase;
        const uint32_t fin = finish(raw, wbase + 3);       // becomes word (wbase+1)+2
        const uint32_t idx = wbase + 4u;
        const bool fetch = cross & ((int)end_byte - (int)(4u * idx) > 0);
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
        low = st[0];
        r = st[1] - st[0];
        dv = st[2] - st[0];
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

// CDF row held by a warp.  EPL = 8: lane l holds entries 8l..8l+7 (two per register) plus the first
// entry of lane l+1; EPL = 1: lane l holds entry l.  Padding entries (index >= L) are stored as 0.
template <int EPL>
struct RowRegs;
template <>
struct RowRegs<8> {
    uint4 v;
    __device__ __forceinline__ void load(const uint16_t *row, int lane) {
        v = __ldg(reinterpret_cast<const uint4 *>(row) + lane);
    }
};
template <>
struct RowRegs<1> {
    uint32_t v;
    __device__ __forceinline__ void load(const uint16_t *row, int lane) { v = (uint32_t)__ldg(row + lane); }
};

__device__ __forceinline__ bool below(uint32_t e, uint32_t r, uint64_t target) {   // e * (r+1) < target
    return ((uint64_t)r * e + e) < target;
}

// Search the row for the symbol whose interval contains the code value.  Returns the symbol and
// its bounds: c_lo = cdf[sym], c_hi = cdf[sym+1] (2^16 for the last symbol).
//   reference: count = ((value-low+1)*2^16-1)/span; sym = largest m with cdf[m] <= count, floor 0
//   here:      cdf[m] <= count  <=>  cdf[m]*span < (value-low+1)<<16      (no division)
template <bool FULLROW>
__device__ __forceinline__ int search_row(const RowRegs<8> &row, uint32_t r, uint64_t target, int lane, int L,
                                          uint32_t &c_lo, uint32_t &c_hi) {
    // every lane tests its 8 entries; rows are non-decreasing, so cdf[sym] is the largest "true" entry
    // and cdf[sym+1] the smallest "false" one: two warp reductions (REDUX) + one for the index
    const uint32_t w[4] = {row.v.x, row.v.y, row.v.z, row.v.w};
    uint32_t lane_lo = 0u, lane_hi = 0x10000u;
    int n_true = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t e = (j & 1) ? (w[j >> 1] >> 16) : (w[j >> 1] & 0xFFFFu);
        const bool valid = FULLROW || (lane * 8 + j) < L;         // padding entries are never true
        const bool f = ((lane | j) == 0) || (valid && below(e, r, target));
        lane_lo = f ? max(lane_lo, e) : lane_lo;
        lane_hi = (f || !valid) ? lane_hi : min(lane_hi, e);
        n_true += f ? 1 : 0;
    }
    c_lo = __reduce_max_sync(FULL, lane_lo);
    c_hi = __reduce_min_sync(FULL, lane_hi);
    return __reduce_add_sync(FULL, n_true) - 1;
}

template <bool FULLROW>
__device__ __forceinline__ int search_row(const RowRegs<1> &row, uint32_t r, uint64_t target, int lane, int L,
                                          uint32_t &c_lo, uint32_t &c_hi) {
    const bool f = (lane == 0) || ((lane < L) && below(row.v, r, target));
    const int n = __popc(__ballot_sync(FULL, f));
    const int sym = n - 1;
    c_lo = __shfl_sync(FULL, row.v, sym);
    const uint32_t nxt = __shfl_sync(FULL, row.v, n & 31);
    c_hi = (n >= L) ? 0x10000u : nxt;
    return sym;
}

// one symbol: search, update [low, high], renormalise, shift code bits into `value`
template <int EPL, bool FULLROW>
__device__ __forceinline__ int decode_step(const RowRegs<EPL> &cur, CoderState &cs, BitSource &src, int lane, int L,
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
    uint32_t c_lo, c_hi;
    const int sym = search_row<FULLROW>(cur, r_cmp, target, lane, L, c_lo, c_hi);
    if (update) cs.update(c_lo, c_hi, src);
    return sym;
}

template <int EPL, bool FULLROW>
__global__ void __launch_bounds__(32 * DEC_WARPS_PER_CTA)
ac_decode_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, int L,
                 uint32_t first, uint32_t count) {
    constexpr int D = 8;   // row prefetch distance (symbols)
    const int sid = blockIdx.x * DEC_WARPS_PER_CTA + (threadIdx.x >> 5);
    if (sid >= n_streams) return;
    const int lane = threadIdx.x & 31;
    const l3c_dec_stream_t st = streams[sid];
    const uint32_t n = st.n_sym;
    if (first >= n) return;
    const uint32_t last = (count > n - first) ? n : first + count;   // exclusive

    BitSource src;
    const uint32_t bit0 = src.open(st.in, st.in_len);

    CoderState cs;
    if (first == 0) {
        src.seek(bit0);
        cs.reset(src.take(32));
    } else {
        cs.restore(st.state);
        src.seek(st.state[3] + bit0);
    }

    const uint16_t *__restrict__ table = st.table;
    const int64_t pitch = st.row_pitch;
    uint8_t *__restrict__ sym_out = st.sym_out;
    const bool vec_out = ((reinterpret_cast<uintptr_t>(sym_out) | first) & 3u) == 0u;

    // symbols handled by the unrolled main loop: whole groups of D, never the stream's final symbol
    const uint32_t upd_end = (last == n) ? n - 1 : last;          // symbols < upd_end update the state
    const uint32_t main_end = first + ((upd_end - first) / D) * D;

    RowRegs<EPL> ring[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const uint32_t i = first + d;
        if (i < last) ring[d].load(table + (int64_t)i * pitch, lane);
    }
    uint32_t base = first;
    for (; base < main_end; base += D) {
        uint32_t packed[D / 4];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            const uint32_t i = base + d;
            const RowRegs<EPL> cur = ring[d];
            if (i + D < last) ring[d].load(table + (int64_t)(i + D) * pitch, lane);
            const int sym = decode_step<EPL, FULLROW>(cur, cs, src, lane, L, true);
            if ((d & 3) == 0) packed[d >> 2] = 0u;
            packed[d >> 2] |= (uint32_t)sym << (8 * (d & 3));
            if (!vec_out && lane == 0) sym_out[i] = (uint8_t)sym;
        }
        if (vec_out && lane == 0) {
#pragma unroll
            for (int q = 0; q < D / 4; ++q) *reinterpret_cast<uint32_t *>(sym_out + base + 4 * q) = packed[q];
        }
    }
    // tail (< D symbols, may contain the final symbol, which leaves the state untouched:
    // torchac.cpp:335-337)
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const uint32_t i = base + d;
        if (i < last) {
            const int sym = decode_step<EPL, FULLROW>(ring[d], cs, src, lane, L, i < upd_end);
            if (lane == 0) sym_out[i] = (uint8_t)sym;
        }
    }

    if (lane == 0 && st.state != nullptr) {
        cs.save(st.state);
        st.state[3] = src.pos - bit0;
    }
}

// ---------------------------------------------------------------------------------------------
// decoder, alphabets of at most 32 symbols (bottleneck and uniform-prior streams): one CDF entry per
// lane, ballot + popc + two shuffles.  Groups of 8 symbols run as straight-line speculative code
// (see v3::ac_decode256_kernel); a group that trips the sticky flag is replayed with decode_step().
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * DEC_WARPS_PER_CTA)
ac_decode32_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, int L,
                   uint32_t first, uint32_t count) {
    constexpr int D = 8;   // symbols per group = row prefetch distance
    const int sid = blockIdx.x * DEC_WARPS_PER_CTA + (threadIdx.x >> 5);
    if (sid >= n_streams) return;
    const int lane = threadIdx.x & 31;
    const l3c_dec_stream_t st = streams[sid];
    const uint32_t n = st.n_sym;
    if (first >= n) return;
    const uint32_t last = (count > n - first) ? n : first + count;   // exclusive

    BitSource src;
    const uint32_t bit0 = src.open(st.in, st.in_len);
    CoderState cs;
    if (first == 0) {
        src.seek(bit0);
        cs.reset(src.take(32));
    } else {
        cs.restore(st.state);
        src.seek(st.state[3] + bit0);
    }

    const uint16_t *__restrict__ table = st.table;
    const int64_t pitch = st.row_pitch;
    uint8_t *__restrict__ sym_out = st.sym_out;
    const bool vec_out = ((reinterpret_cast<uintptr_t>(sym_out) | first) & 3u) == 0u;
    const bool in_row = lane < L;

    const uint32_t upd_end = (last == n) ? n - 1 : last;          // symbols < upd_end update the state
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
                if (lane == 0) {
                    if (vec_out) {
#pragma unroll
                        for (int q = 0; q < D / 4; ++q)
                            *reinterpret_cast<uint32_t *>(sym_out + base + 4 * q) = packed[q];
                    } else {
#pragma unroll
                        for (int d = 0; d < D; ++d) sym_out[base + d] = (uint8_t)(packed[d >> 2] >> (8 * (d & 3)));
                    }
                }
                continue;
            }
            cs = cs0;                 // replay this group exactly (the ring already holds the next group's rows)
            src = src0;
        }
#pragma unroll 1
        for (int d = 0; d < D; ++d) {
            const uint32_t i = base + d;
            RowRegs<1> cur;
            cur.load(table + (int64_t)i * pitch, lane);
            const int sym = decode_step<1, false>(cur, cs, src, lane, L, true);
            if (lane == 0) sym_out[i] = (uint8_t)sym;
        }
    }
    // tail (< D symbols, may contain the stream's final symbol, which leaves the state untouched:
    // torchac.cpp:335-337)
#pragma unroll 1
    for (uint32_t i = base; i < last; ++i) {
        RowRegs<1> cur;
        cur.load(table + (int64_t)i * pitch, lane);
        const int sym = decode_step<1, false>(cur, cs, src, lane, L, i < upd_end);
        if (lane == 0) sym_out[i] = (uint8_t)sym;
    }

    if (lane == 0 && st.state != nullptr) {
        cs.save(st.state);
        st.state[3] = src.pos - bit0;
    }
}

// ---------------------------------------------------------------------------------------------
// decoder, 256-symbol alphabets (the RGB streams): CTA = decoder warp + helper warp per stream
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

template <int SPC>
__global__ void __launch_bounds__(64 * SPC)
ac_decode256_kernel(const l3c_dec_stream_t *__restrict__ streams, int n_streams, uint32_t first, uint32_t count) {
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
    const uint32_t n = st.n_sym;
    if (first >= n) return;
    const uint32_t last = (count > n - first) ? n : first + count;   // exclusive
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
                uint32_t pack0 = 0u, pack1 = 0u;
#pragma unroll
                for (int d = 0; d < G; ++d) {
                    if (ibase + d < last) {
                        const uint32_t top = tops[g * G + d];
                        const uint4 a = ring[g * G + d][0][lane];
                        const uint4 b = ring[g * G + d][1][lane];
                        int c = (a.x <= top) + (a.y <= top) + (a.z <= top) + (a.w <= top) + (b.x <= top) + (b.y <= top) +
                                (b.z <= top) + (b.w <= top);
                        int tot = __reduce_add_sync(FULL, c);
                        tot = tot > 0 ? tot - 1 : 0;
                        if (d < 4) pack0 |= (uint32_t)tot << (8 * d);
                        else pack1 |= (uint32_t)tot << (8 * (d - 4));
                    }
                }
                if (lane == 0) {
                    const bool vec = ((reinterpret_cast<uintptr_t>(sym_out) | ibase) & 3u) == 0u && ibase + G <= last;
                    if (vec) {
                        *reinterpret_cast<uint32_t *>(sym_out + ibase) = pack0;
                        *reinterpret_cast<uint32_t *>(sym_out + ibase + 4) = pack1;
                    } else {
                        for (int d = 0; d < G; ++d)
                            if (ibase + d < last)
                                sym_out[ibase + d] = (uint8_t)(((d < 4 ? pack0 : pack1) >> (8 * (d & 3))) & 0xFFu);
                    }
                }
                __syncwarp();
            }
            if (gi < n_groups) {
#pragma unroll
                for (int d = 0; d < G; ++d) {
                    const uint4 v = cur[d];
                    uint32_t nx = __shfl_down_sync(FULL, v.x, 1);
                    if (lane == 31) nx = 0u;                                  // row end -> upper bound 2^16
                    uint4 lo, hi;
                    // proposal of entry m: (cdf[m] << 16) | ((cdf[m+1] - 1) & 0xFFFF)
                    lo.x = (v.x << 16) | (((v.x >> 16) - 1u) & 0xFFFFu);
                    lo.y = (v.x & 0xFFFF0000u) | (((v.y & 0xFFFFu) - 1u) & 0xFFFFu);
                    lo.z = (v.y << 16) | (((v.y >> 16) - 1u) & 0xFFFFu);
                    lo.w = (v.y & 0xFFFF0000u) | (((v.z & 0xFFFFu) - 1u) & 0xFFFFu);
                    hi.x = (v.z << 16) | (((v.z >> 16) - 1u) & 0xFFFFu);
                    hi.y = (v.z & 0xFFFF0000u) | (((v.w & 0xFFFFu) - 1u) & 0xFFFFu);
                    hi.z = (v.w << 16) | (((v.w >> 16) - 1u) & 0xFFFFu);
                    hi.w = (v.w & 0xFFFF0000u) | (((nx & 0xFFFFu) - 1u) & 0xFFFFu);
                    ring[g * G + d][0][lane] = lo;
                    ring[g * G + d][1][lane] = hi;
                }
                mbar_arrive(bar0 + 8 * g);                                    // full[g]
            }
        }
        return;
    }

    // ============================ decoder warp ============================
    BitSource src;
    const uint32_t bit0 = src.open(st.in, st.in_len);
    CoderState cs;
    if (first == 0) {
        src.seek(bit0);
        cs.reset(src.take(32));
    } else {
        cs.restore(st.state);
        src.seek(st.state[3] + bit0);
    }
    const uint32_t upd_end = (last == n) ? n - 1u : last;                     // symbols < upd_end update the state
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
                const uint32_t r = cs.r;
                const uint32_t dv = cs.dv;
                uint64_t target = ((uint64_t)dv + 1ull) << 16;
                uint32_t r_cmp = r;
                if (dv > r) {                                                 // corrupt / foreign input only
                    target = (uint64_t)foreign_count16(cs.low + dv, cs.low, r) + 1ull;
                    r_cmp = 0u;
                }
                const uint32_t pk[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                uint32_t best = 0u;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const bool fj = ((lane | j) == 0) || below(pk[j] >> 16, r_cmp, target);
                    best = fj ? max(best, pk[j]) : best;
                }
                const uint32_t top = __reduce_max_sync(FULL, best);
                if (lane == 0) tops[g * G + d] = top;
                if (i != n - 1)                                               // torchac.cpp:335-337
                    cs.update(top >> 16, (top & 0xFFFFu) + 1u, src);
            }
        }
        __syncwarp();
        mbar_arrive(bar0 + 16 + 8 * g);                                       // empty[g]
    }
    if (lane == 0 && st.state != nullptr) {
        cs.save(st.state);
        st.state[3] = src.pos - bit0;
    }
}

}  // namespace v3

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
        const uint32_t b1 = (uint32_t)min(b0 + (uint64_t)PACK_CHUNK, (uint64_t)len);
        for (uint32_t i = (uint32_t)b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = st.out[i];
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
extern "C" int l3c_ac_encode_streams(const l3c_enc_stream_t *streams_dev, int n_streams,
                                     uint32_t *out_len_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_encode_streams: n_streams=%d", n_streams);
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && out_len_dev, "l3c_ac_encode_streams: null pointer");
    const int grid = ceil_div(n_streams, ENC_WARPS_PER_CTA);
    ac_encode_kernel<<<grid, 32 * ENC_WARPS_PER_CTA, 0, (cudaStream_t)stream>>>(
        streams_dev, n_streams, out_len_dev);
    L3C_LAUNCH_CHECK("ac_encode_kernel");
    return L3C_OK;
}

namespace l3c {
std::atomic<int> g_dec_spc{0};   // l3c_set_decoder_streams_per_cta: 0 = L3C_DEC_SPC / the default
}

extern "C" int l3c_set_decoder_streams_per_cta(int spc) {
    L3C_REQUIRE(spc == 0 || spc == 1 || spc == 2 || spc == 4,
                "l3c_set_decoder_streams_per_cta: spc=%d not in {0, 1, 2, 4}", spc);
    l3c::g_dec_spc.store(spc);
    return L3C_OK;
}

extern "C" int l3c_ac_decode_streams(const l3c_dec_stream_t *streams_dev, int n_streams, int L,
                                     uint32_t first, uint32_t count, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(n_streams >= 0, "l3c_ac_decode_streams: n_streams=%d", n_streams);
    L3C_REQUIRE(L >= 1 && L <= 256, "l3c_ac_decode_streams: L=%d not in [1,256]", L);
    if (n_streams == 0 || count == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev, "l3c_ac_decode_streams: null pointer");
    const int grid = ceil_div(n_streams, DEC_WARPS_PER_CTA);
    const dim3 blk(32 * DEC_WARPS_PER_CTA);
    cudaStream_t st = (cudaStream_t)stream;
    if (L <= 32) {
        ac_decode32_kernel<<<grid, blk, 0, st>>>(streams_dev, n_streams, L, first, count);
    } else if (L == 256) {
        static const int env_spc = [] {
            const char *e = getenv("L3C_DEC_SPC");
            const int v = e ? atoi(e) : 1;
            return (v == 1 || v == 2 || v == 4) ? v : 1;
        }();
        static bool configured_dev[64] = {};
        const int forced = g_dec_spc.load(std::memory_order_relaxed);
        const int spc = forced ? forced : env_spc;
        bool &configured = configured_dev[current_device_slot()];
        if (!configured) {
            L3C_CUDA(cudaFuncSetAttribute(v3::ac_decode256_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          4 * v3::STREAM_SMEM));
            configured = true;
        }
        if (spc == 4)
            v3::ac_decode256_kernel<4><<<ceil_div(n_streams, 4), 256, 4 * v3::STREAM_SMEM, st>>>(streams_dev, n_streams, first, count);
        else if (spc == 2)
            v3::ac_decode256_kernel<2><<<ceil_div(n_streams, 2), 128, 2 * v3::STREAM_SMEM, st>>>(streams_dev, n_streams, first, count);
        else
            v3::ac_decode256_kernel<1><<<n_streams, 64, v3::STREAM_SMEM, st>>>(streams_dev, n_streams, first, count);
    } else {
        ac_decode_kernel<8, false><<<grid, blk, 0, st>>>(streams_dev, n_streams, L, first, count);
    }
    L3C_LAUNCH_CHECK("ac_decode_kernel");
    return L3C_OK;
}

extern "C" int l3c_pack_streams(const l3c_enc_stream_t *streams_dev, const uint32_t *len_dev,
                                const uint64_t *dst_off_dev, int n_streams, uint8_t *blob_dev,
                                void *stream) {
    using namespace l3c;
    if (n_streams == 0) return L3C_OK;
    L3C_REQUIRE(streams_dev && len_dev && dst_off_dev && blob_dev && n_streams > 0 && n_streams <= 65535,
                "l3c_pack_streams: bad arguments");
    dim3 grid(PACK_GRID_X, n_streams);
    pack_streams_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(streams_dev, len_dev, dst_off_dev, blob_dev);
    L3C_LAUNCH_CHECK("pack_streams_kernel");
    return L3C_OK;
}

extern "C" int l3c_lut_intervals(const uint8_t *sym_dev, const uint32_t *lut_dev, int64_t n,
                                 uint32_t *intervals_dev, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(sym_dev && lut_dev && intervals_dev && n >= 0, "l3c_lut_intervals: bad arguments");
    if (n == 0) return L3C_OK;
    lut_intervals_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(sym_dev, lut_dev, n,
                                                                                       intervals_dev);
    L3C_LAUNCH_CHECK("lut_intervals_kernel");
    return L3C_OK;
}
