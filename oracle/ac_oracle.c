/*
 * oracle/ac_oracle.c -- TEST INFRASTRUCTURE ONLY (CPU oracle).
 *
 * A plain-C restatement of the reference's entropy-coding arithmetic, used by tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline leg as the *checker* for the CUDA
 * path.  Nothing under l3c_pytorch_b200/ may call into this file.
 *
 * What it restates (file:line in /root/reference):
 *   - the 32-bit-state / 16-bit-precision binary arithmetic ENCODER
 *       src/torchac/torchac_backend/torchac.cpp:152-227  (+ bit packer :63-93)
 *   - the matching DECODER with its per-row binary search
 *       src/torchac/torchac_backend/torchac.cpp:276-381  (+ bit reader :96-128)
 *   - the logistic-mixture CDF table formula of the reference CUDA kernel
 *       src/torchac/torchac_backend/torchac_kernel.cu:16-76
 *
 * Pinning: oracle/pin_oracle.py checks these functions byte-for-byte against the reference's
 * own torchac.cpp compiled unmodified into oracle/_ref/ (KATs of SURVEY.md §8c + random tables);
 * tests/test_oracle_kat.py re-checks the committed known-answer vectors on every run.
 *
 * Conventions: a CDF "row" has Lp = L+1 uint16 entries; row i starts at cdf + i*row_stride
 * (row_stride == 0 means one shared row, e.g. the uniform prior).  The last entry of a row
 * is never read: the upper bound of the top symbol is the constant 2^16.
 */
#include <stdint.h>
#include <stddef.h>
#include <math.h>

#define AC_PRECISION 16
#define AC_TOP 0x10000u
#define AC_HALF 0x80000000u
#define AC_QUARTER 0x40000000u
#define AC_THREE_QUARTER 0xC0000000u

/* ---- MSB-first bit sink (torchac.cpp:63-93) ------------------------------------------- */
typedef struct {
    uint8_t *buf;
    size_t cap;
    size_t n;        /* bytes produced so far (may exceed cap: then nothing more is stored) */
    uint8_t acc;
    int nacc;
} bitsink_t;

static void sink_bit(bitsink_t *s, int bit) {
    s->acc = (uint8_t)((s->acc << 1) | (bit & 1));
    if (++s->nacc == 8) {
        if (s->n < s->cap) s->buf[s->n] = s->acc;
        s->n++;
        s->nacc = 0;
        s->acc = 0;
    }
}

static void sink_bit_then_inverse(bitsink_t *s, int bit, uint64_t *pending) {
    sink_bit(s, bit);
    while (*pending) {
        sink_bit(s, !bit);
        (*pending)--;
    }
}

/* ---- encoder (torchac.cpp:152-227) ------------------------------------------------------ */
size_t oracle_ac_encode(const uint16_t *cdf, int64_t row_stride, int n_sym, int Lp,
                        const int16_t *sym, uint8_t *out, size_t out_cap) {
    bitsink_t sink = {out, out_cap, 0, 0, 0};
    uint32_t low = 0, high = 0xFFFFFFFFu;
    uint64_t pending = 0;
    const int top_symbol = Lp - 2;

    for (int i = 0; i < n_sym; ++i) {
        const uint16_t *row = cdf + (int64_t)i * row_stride;
        const int s = sym[i];
        const uint64_t span = (uint64_t)high - (uint64_t)low + 1u;
        const uint32_t c_lo = row[s];
        const uint32_t c_hi = (s == top_symbol) ? AC_TOP : row[s + 1];

        high = (low - 1u) + (uint32_t)((span * (uint64_t)c_hi) >> AC_PRECISION);
        low = low + (uint32_t)((span * (uint64_t)c_lo) >> AC_PRECISION);

        for (;;) {
            if (high < AC_HALF) {
                sink_bit_then_inverse(&sink, 0, &pending);
            } else if (low >= AC_HALF) {
                sink_bit_then_inverse(&sink, 1, &pending);
            } else if (low >= AC_QUARTER && high < AC_THREE_QUARTER) {
                pending++;
                low = (low << 1) & 0x7FFFFFFFu;
                high = (high << 1) | 0x80000001u;
                continue;
            } else {
                break;
            }
            low <<= 1;
            high = (high << 1) | 1u;
        }
    }

    /* termination: one disambiguating bit (+ whatever underflow bits are still owed) */
    pending += 1;
    sink_bit_then_inverse(&sink, low < AC_QUARTER ? 0 : 1, &pending);
    while (sink.nacc != 0) sink_bit(&sink, 0);   /* zero-pad to a whole byte */
    return sink.n;
}

/* ---- MSB-first bit source, zero-filled past the end (torchac.cpp:96-128) ----------------- */
typedef struct {
    const uint8_t *buf;
    size_t len;
    size_t pos;
    uint8_t cur;
    int left;
} bitsrc_t;

static void src_shift_in(bitsrc_t *b, uint32_t *value) {
    if (b->left == 0) {
        if (b->pos == b->len) {
            *value <<= 1;
            return;
        }
        b->cur = b->buf[b->pos++];
        b->left = 8;
    }
    *value = (*value << 1) | ((uint32_t)(b->cur >> (b->left - 1)) & 1u);
    b->left--;
}

/* binary search exactly as the reference walks it (torchac.cpp:276-296) */
static uint16_t row_search(const uint16_t *row, uint16_t target, uint16_t top_symbol) {
    uint16_t left = 0;
    uint16_t right = (uint16_t)(top_symbol + 1);
    while (left + 1 < right) {
        const uint16_t mid = (uint16_t)((left + right) / 2);
        const uint16_t v = row[mid];
        if (v < target) {
            left = mid;
        } else if (v > target) {
            right = mid;
        } else {
            return mid;
        }
    }
    return left;
}

/* ---- decoder (torchac.cpp:299-381) --------------------------------------------------------
 * trace (may be NULL): 4 words per symbol, trace[4*i ..] = (low, high, value, code bits read)
 * when symbol i is reached -- the coder state a decoder resumed at symbol i starts from. */
void oracle_ac_decode_trace(const uint16_t *cdf, int64_t row_stride, int n_sym, int Lp,
                            const uint8_t *in, size_t in_len, int16_t *out, uint32_t *trace) {
    bitsrc_t src = {in, in_len, 0, 0, 0};
    uint32_t low = 0, high = 0xFFFFFFFFu, value = 0;
    uint32_t nbits = 32;
    const int top_symbol = Lp - 2;

    for (int i = 0; i < 32; ++i) src_shift_in(&src, &value);

    for (int i = 0; i < n_sym; ++i) {
        if (trace) {
            trace[4 * (size_t)i + 0] = low;
            trace[4 * (size_t)i + 1] = high;
            trace[4 * (size_t)i + 2] = value;
            trace[4 * (size_t)i + 3] = nbits;
        }
        const uint16_t *row = cdf + (int64_t)i * row_stride;
        const uint64_t span = (uint64_t)high - (uint64_t)low + 1u;
        const uint16_t count =
            (uint16_t)((((uint64_t)value - (uint64_t)low + 1u) * (uint64_t)AC_TOP - 1u) / span);
        const uint16_t s = row_search(row, count, (uint16_t)top_symbol);
        out[i] = (int16_t)s;
        if (i == n_sym - 1) break;

        const uint32_t c_lo = row[s];
        const uint32_t c_hi = (s == top_symbol) ? AC_TOP : row[s + 1];
        high = (low - 1u) + (uint32_t)((span * (uint64_t)c_hi) >> AC_PRECISION);
        low = low + (uint32_t)((span * (uint64_t)c_lo) >> AC_PRECISION);

        for (;;) {
            if (low >= AC_HALF || high < AC_HALF) {
                low <<= 1;
                high = (high << 1) | 1u;
            } else if (low >= AC_QUARTER && high < AC_THREE_QUARTER) {
                low = (low << 1) & 0x7FFFFFFFu;
                high = (high << 1) | 0x80000001u;
                value -= AC_QUARTER;
            } else {
                break;
            }
            src_shift_in(&src, &value);
            nbits++;
        }
    }
}

void oracle_ac_decode(const uint16_t *cdf, int64_t row_stride, int n_sym, int Lp,
                      const uint8_t *in, size_t in_len, int16_t *out) {
    oracle_ac_decode_trace(cdf, row_stride, n_sym, Lp, in, in_len, out, NULL);
}

/* ---- logistic-mixture CDF table (torchac_kernel.cu:16-76) --------------------------------
 * params are [K][N] row-major fp32 (a 1xKxHxW tensor flattened), targets has Lp entries.
 * cdf[n*Lp + l] = (uint16) ( lrintf( sum_k pi[k][n]*sigmoid((t_l - mu[k][n]) * exp(-logs[k][n]))
 *                                    * (65536 - (Lp-1)) ) + l )
 * The sigmoid is evaluated as 1.0/(1.0+expf(-a)) with the double-typed literals of the
 * reference (torchac_kernel.cu:16-18) and rounded back to float.
 */
static float ref_sigmoidf(float a) { return (float)(1.0 / (1.0 + (double)expf(-a))); }

void oracle_mixture_cdf(const float *targets, const float *means, const float *log_scales,
                        const float *probs, int K, int N, int Lp, uint16_t *cdf_out) {
    const float scale = (float)(AC_TOP - (uint32_t)(Lp - 1));
    for (int n = 0; n < N; ++n) {
        for (int l = 0; l < Lp; ++l) {
            float acc = 0.f;
            for (int k = 0; k < K; ++k) {
                const float inv_s = expf(-log_scales[(size_t)k * N + n]);
                const float centred = targets[l] - means[(size_t)k * N + n];
                acc += probs[(size_t)k * N + n] * ref_sigmoidf(centred * inv_s);
            }
            cdf_out[(size_t)n * Lp + l] = (uint16_t)(lrintf(acc * scale) + l);
        }
    }
}
