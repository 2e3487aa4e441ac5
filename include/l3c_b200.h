/*
 * l3c_b200.h -- C ABI of libl3c_b200.so: the sm_90a implementation of L3C's encode/decode hot path.
 *
 * Plain pointers and sizes only (no torch types).  Every entry point returns 0 on success or a
 * negative L3C_E* code; l3c_last_error() gives the message of the last failure on the calling
 * thread.  "dev" pointers are CUDA device pointers on the current device, "host" pointers are
 * ordinary (ideally pinned) host memory.  `stream` is a cudaStream_t passed as void* (NULL = the
 * legacy default stream).  Kernels are asynchronous on `stream` unless a function says it
 * synchronises.
 *
 * Section A are the drop-in replacements for the FIVE exports of the reference's native module
 * (pybind module torchac_backend_{cpu,gpu}: /root/reference/src/torchac/torchac_backend/
 * torchac.cpp:433-443).  Sections B..E are the batched, device-resident building blocks the host
 * mirror (l3c_pytorch_b200.*) composes into the reference's Bitcoding / MultiscaleBlueprint API;
 * section F adds the ones the batched torchac calls compose with section B.
 *
 * Layout conventions
 *   activations ........ NHWC fp32, channel pitch given explicitly where slices are written
 *   conv weights ....... [KH][KW][Cin][CoutPad] fp32 (host mirror repacks the reference's OIHW)
 *   symbol planes ...... uint8  [N][C][H*W]    (one plane = one coded stream, row-major H,W;
 *                                               flatten order of coders.py:49-50)
 *   intervals .......... uint32 [N][C][H*W]    c_low | (c_high-1) << 16
 *   CDF tables ......... uint16 rows of `pitch` entries (entries 0..L-1 used; the reference's
 *                        (L+1)-th entry is never read, torchac.cpp:181,280)
 */
#ifndef L3C_B200_H_
#define L3C_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define L3C_OK 0
#define L3C_EINVAL (-1)   /* bad argument (shape/alignment/range)      -> reference raises RuntimeError */
#define L3C_ECUDA (-2)    /* CUDA runtime error                                                          */
#define L3C_EOVERFLOW (-3)/* output buffer too small                                                     */
#define L3C_ENODEV (-4)   /* no sm_90 device                                                            */
#define L3C_EUNSUPPORTED (-5) /* optional facility not offered by this driver (caller may do without)      */

const char *l3c_last_error(void);
int l3c_version(void);

/* Launch log (no reference counterpart; evidence plumbing): every kernel this library launches is
 * counted under its kernel name.  Writes "kernel_name count\n" lines into buf (truncated to cap, may be
 * NULL) and returns the TOTAL number of launches since the last reset; reset != 0 clears the counters. */
long long l3c_launch_log(char *buf, size_t cap, int reset);

/* ------------------------------------------------------------------------------------------
 * A. Drop-in native exports (reference: torchac.cpp:433-443; python shim torchac.py:87-166)
 * ---------------------------------------------------------------------------------------- */

/* The four coding functions accept every Lp in [2, 32769] (L = Lp - 1 symbols, int16 symbols as in the reference);
 * any other Lp is L3C_EINVAL.  Rows must be strictly increasing over entries 0..L-1, as the reference's binary
 * search assumes; the last entry is never read.
 *
 * replaces `cuda_supported()` (torchac.cpp:439,441): 1 iff an sm_90 device is usable. */
int l3c_cuda_supported(void);

/* replaces `encode_cdf(cdf, sym) -> bytes` (torchac.cpp:262-269 -> encode() :152-227).
 * cdf_host: int16/uint16 [n_sym][Lp] (the 1HWLp tensor, flattened); sym_host: int16 [n_sym].
 * Synchronous.  *out_len receives the byte count; L3C_EOVERFLOW if it exceeds out_cap. */
int l3c_encode_cdf(const uint16_t *cdf_host, int64_t n_sym, int Lp, const int16_t *sym_host,
                   uint8_t *out_host, size_t out_cap, size_t *out_len);

/* replaces `decode_cdf(cdf, in) -> int16 tensor` (torchac.cpp:424-430 -> decode() :299-381).
 * n_sym comes from the cdf shape, exactly as in the reference; short input is zero-filled. */
int l3c_decode_cdf(const uint16_t *cdf_host, int64_t n_sym, int Lp, const uint8_t *in_host,
                   size_t in_len, int16_t *sym_out_host);

/* replaces `encode_logistic_mixture(targets, means, log_scales, logit_probs_softmax, sym)`
 * (torchac.cpp:231-258; CDF formula torchac_kernel.cu:20-76).  targets_dev f32[Lp];
 * means/log_scales/probs_dev f32 [K][n_sym] (1KHW contiguous, CUDA); sym_host int16 (CPU, as in
 * the reference).  No CDF table is materialised: only the two bounds of each coded symbol are
 * evaluated.  Synchronous.
 * log_scales are used as given, unclamped, as the reference's torchac does.  Below about -88 the
 * scale factor exp(-log_scale) overflows to inf.  An entry whose target then equals a component's
 * mean evaluates to NaN and becomes cdf[l] = l, which can make the row decrease there and leave a
 * symbol without an interval.  The reference's callers clamp log-scales at -7
 * (logistic_mixture.py:57), which is far from this limit. */
int l3c_encode_logistic_mixture(const float *targets_dev, const float *means_dev,
                                const float *log_scales_dev, const float *probs_dev, int K,
                                int64_t n_sym, int Lp, const int16_t *sym_host,
                                uint8_t *out_host, size_t out_cap, size_t *out_len);

/* replaces `decode_logistic_mixture(..., in) -> int16 tensor` (torchac.cpp:385-421). */
int l3c_decode_logistic_mixture(const float *targets_dev, const float *means_dev,
                                const float *log_scales_dev, const float *probs_dev, int K,
                                int64_t n_sym, int Lp, const uint8_t *in_host, size_t in_len,
                                int16_t *sym_out_host);

/* ------------------------------------------------------------------------------------------
 * B. Range coder, batched: one warp per stream, any number of streams per launch
 *    (reference loop: torchac.cpp:174-207 encode, :325-373 decode, one stream per call)
 * ---------------------------------------------------------------------------------------- */

typedef struct {
    const uint32_t *intervals;  /* dev: n_sym packed intervals                                  */
    uint8_t *out;               /* dev: output slot, 4-byte aligned, out_cap bytes              */
    uint32_t n_sym;
    uint32_t out_cap;           /* multiple of 4                                                */
} l3c_enc_stream_t;

/* out_len_dev[i] = bytes produced by stream i (if > out_cap the slot content is truncated; a stream of 2^32 bytes or
 * more reports 2^32 - 1).  out_len is unsigned: read it as uint32, not int32. */
int l3c_ac_encode_streams(const l3c_enc_stream_t *streams_dev, int n_streams,
                          uint32_t *out_len_dev, void *stream);

typedef struct {
    const uint16_t *table;      /* dev: CDF rows for symbols [0, n_sym) of this stream           */
    const uint8_t *in;          /* dev: code bytes at ANY byte address (decoded in place from the  */
                                /*      container); the buffer must be readable 4 bytes past the end */
    uint8_t *sym_out;           /* dev: n_sym decoded symbols, uint8; for L > 256 n_sym           */
                                /*      little-endian uint16, 2-byte aligned.  Nothing past n_sym  */
                                /*      symbols is written.                                       */
    uint32_t *state;            /* dev: coder state (low, high, value, code bits read); lets one  */
                                /*      stream be decoded in several launches (chunks).  4 words, */
                                /*      word 3 the low 32 bits of the bits read; a stream with    */
                                /*      in_len >= 2^28 takes a 5th word, their high 32 bits.  A    */
                                /*      shorter stream read 2^32 bits or more, far past its end,  */
                                /*      sets bit 31 of word 0 (low is below 2^31)                 */
    int64_t row_pitch;          /* entries between consecutive rows; 0 = one shared row.  Every   */
                                /*      row is read whole: 32 entries for L <= 32, 256 for L <= 256,*/
                                /*      round_up(L, 8) for L > 256, 16-byte aligned.  Entries past */
                                /*      L may hold anything.  For L > 256 the pitch must be 0 or a */
                                /*      multiple of 8 that is >= L.                               */
    uint32_t n_sym;             /* total symbols of the stream                                    */
    uint32_t in_len;
} l3c_dec_stream_t;

/* Decodes symbols [first, first+count) of every stream (count clipped to n_sym).  first == 0
 * initialises the coder state from the stream head, otherwise it is resumed from `state`.
 * L = number of symbols of the alphabet, 1 to 32768.  For L > 256 the descriptors are first copied to the host and
 * checked (row_pitch, 16-byte aligned table, 2-byte aligned sym_out; L3C_EINVAL otherwise), so the call waits for
 * `stream`. */
int l3c_ac_decode_streams(const l3c_dec_stream_t *streams_dev, int n_streams, int L,
                          uint32_t first, uint32_t count, void *stream);

/* Seek points (DESIGN §4.13).  A seek point of a stream is the decoder's state before one of its symbols j: low, high
 * and the code bits read, 32 + the sum of the renormalisation shifts of the symbols before j (64 bits), plus whether
 * the last of those shifts was an "underflow" shift: then the code value is the last 32 code bits read with bit 31
 * flipped, else those bits.  From a seek point the symbols from j on decode without the ones before it. */

/* l3c_ac_encode_streams, same bytes and lengths, that also records a seek point before symbol j of stream i for
 * j = every, 2 every, ... < n_sym: point j / every - 1 is the 4 words at points_dev[i] + 4 (j / every - 1) =
 * (low, high, bits: low word, bits: high word | underflow flag << 31).  points_dev: device array of n_streams device
 * pointers (a stream with no points may have null).  every: a positive multiple of 32. */
int l3c_ac_encode_streams_seek(const l3c_enc_stream_t *streams_dev, int n_streams, uint32_t *out_len_dev,
                               uint32_t every, uint32_t *const *points_dev, void *stream);

/* Segment decode: every descriptor is one segment of a stream, decoded whole in one launch, all segments in
 * parallel.  table and sym_out point at the segment's first symbol, n_sym is its length, in / in_len the whole
 * stream.  state: null for a segment that starts at the stream's head, else its seek point as 5 words (low, high,
 * flip, bits: low word, bits: high word), flip 0 or 0x80000000 (the underflow flag in bit 31); it is only read.  The
 * segment's final symbol is decoded like any other.  L from 1 to 256 (l3c_ac_decode_streams' rows); larger alphabets
 * are refused (L3C_EINVAL). */
int l3c_ac_decode_segments(const l3c_dec_stream_t *segs_dev, int n_segs, int L, void *stream);

/* l3c_ac_decode_segments for L = 256 whose `table`s point at coarse records (as l3c_ac_decode_streams_coarse). */
int l3c_ac_decode_segments_coarse(const l3c_dec_stream_t *segs_dev, int n_segs, const float *targets_dev,
                                  void *stream);

/* Copies the first min(len_dev[i], out_cap) bytes of encoder slot i (a stream that outgrew its slot is truncated as
 * the slot holds it) to blob_dev + dst_off_dev[i] (byte offsets, any alignment: the final .l3c container layout, so
 * ONE device->host copy returns a whole batch).  Nothing else of the blob is written.  Any number of streams; more
 * than 65535 take several launches. */
int l3c_pack_streams(const l3c_enc_stream_t *streams_dev, const uint32_t *len_dev,
                     const uint64_t *dst_off_dev, int n_streams, uint8_t *blob_dev, void *stream);

/* Assembles the containers of region updates (DESIGN §4.12) in ONE launch from segments seg_host int64 [n_seg][4] =
 * (src, src_off, dst_off, bytes), copying bytes [src_off, src_off + bytes) of a source to out_dev + dst_off:
 *   src 0: old_dev (old_bytes long, the uploaded old containers): a run of unchanged streams with their length fields
 *          and the headers and magics between them;
 *   src 1: slots_dev (slot_bytes long, the encoder slots of the re-encoded streams): one new stream; its length is
 *          also written, as a little-endian u32, to the 4 bytes at out_dev + dst_off - 4.
 * One warp copies each 4 KB chunk of a segment.  The segments and each one's first chunk are copied to seg_dev
 * (device, 8-byte aligned, (5 * n_seg + 1) * 8 bytes) on `stream` before the launch.  Nothing of out_dev outside the
 * destinations is written.  Refused before any GPU work (L3C_EINVAL): null pointers, a source other than 0 or 1, a
 * negative size or (src 1) one of 2^32 bytes or more, a segment outside its source or outside out_dev (length field
 * included), and destinations that overlap (length fields included; an empty segment of src 0 is the point dst_off and
 * is refused strictly inside another destination).  n_seg = 0 does nothing. */
int l3c_splice_streams(const uint8_t *old_dev, int64_t old_bytes, const uint8_t *slots_dev, int64_t slot_bytes,
                       const int64_t *seg_host, int64_t *seg_dev, int n_seg, uint8_t *out_dev, int64_t out_bytes,
                       void *stream);

/* Layout and splice of region updates whose new stream lengths stay in device memory (DESIGN §4.12, "Serving
 * updates").  One stream of a container, in container stream order: */
typedef struct {
    int64_t fixed_off;          /* its offset if every stream of the container had length 0                    */
    int64_t old_off, old_len;   /* where its bytes lie in the old container                                    */
    int64_t src;                /* -1: unchanged; else index i into the call's new lengths, slot_off and caps  */
} l3c_update_stream_t;

/* One container of the call (all int64): */
typedef struct {
    int64_t first_stream, n_streams;  /* its streams: streams_dev[first_stream, first_stream + n_streams)          */
    int64_t fixed_total;              /* its size if every stream had length 0                                     */
    int64_t old_base, old_bytes;      /* the old container at old_dev + old_base, old_bytes long                   */
    int64_t out_base, out_cap;        /* the new one goes to out_dev + out_base and may take up to out_cap bytes    */
    int64_t first_seg, n_new;         /* its n_new re-encoded streams; its 2 n_new + 1 segments at seg_dev +        */
                                      /* 4 first_seg, their chunk prefix at chunk0_dev + first_seg + (its index)   */
} l3c_update_container_t;

/* One CTA per container.  len[s] = old_len[s] for an unchanged stream, new_len_dev[src] for a re-encoded one;
 * new_off[s] = fixed_off[s] + exclusive_scan(len)[s] and the size is fixed_total + sum(len).  Writes the size to
 * info_dev[k] and the container's segments in the form of l3c_splice_streams, int64 [2 n_new + 1][4] =
 * (src, src_off, dst_off, bytes): segment 0 the run of the old container before the first re-encoded stream's
 * length field, then per re-encoded stream j (ascending) its new bytes (src 1, from slot_off_dev[src] of the slots,
 * to out_base + new_off) and the run of the old container after it (src 0, up to the next re-encoded stream's length
 * field or the end).  Runs may be empty.  Offsets are absolute: src_off in the old buffer or the slots, dst_off in the
 * output.  chunk0_dev gets, per container, the exclusive prefix over its segments of l3c_splice_streams_dev's chunks
 * (one per 4 KB of a segment, at least one for src 1) and their total; a container with an error gets no chunks.
 * info_dev[n_containers] is an error flag, zeroed on `stream` first: bit 0 a new length above its cap (the coder
 * clamps its writes to out_cap), bit 1 an inconsistent input (a descriptor outside the arrays, a source index out of
 * range, re-encoded streams other than n_new, a size above out_cap).  L3C_EINVAL for null pointers or negative
 * counts, before any GPU work; n_containers = 0 only clears the flag. */
int l3c_update_layout(const l3c_update_container_t *conts_dev, int n_containers,
                      const l3c_update_stream_t *streams_dev, int64_t n_streams, const int32_t *new_len_dev,
                      const int64_t *slot_off_dev, const int64_t *caps_dev, int64_t n_new,
                      int64_t *seg_dev, int64_t *chunk0_dev, int64_t n_seg, int64_t *info_dev, void *stream);

/* The splice of l3c_splice_streams from the segments l3c_update_layout left in device memory: one warp per 4 KB
 * chunk, grid rows over the containers.  Each segment is checked in the kernel: source 0 or 1, its bytes inside its
 * container's old bytes (src 0) or the slots (src 1, below 2^32), its destination, length field included, inside the
 * container's [out_base, out_base + out_cap) and out_dev.  A segment that fails is not copied and sets bit 1 of
 * *flag_dev.  n_seg: the segments of seg_dev (a container whose segments fall outside them is skipped).  max_chunks: the most chunks a container can have (sizes the grid; any value is correct).  L3C_EINVAL
 * for null pointers or negative counts. */
int l3c_splice_streams_dev(const l3c_update_container_t *conts_dev, int n_containers, const int64_t *seg_dev,
                           const int64_t *chunk0_dev, int64_t n_seg, const uint8_t *old_dev, int64_t old_bytes,
                           const uint8_t *slots_dev, int64_t slot_bytes, uint8_t *out_dev, int64_t out_bytes,
                           int64_t max_chunks, int64_t *flag_dev, void *stream);

/* intervals_dev[i] = lut_dev[sym_dev[i]], i < n -- coding intervals when all pixels share one CDF row
 * (uniform prior of the coarsest scale, bitcoding.py:171-186). lut entry = c_low | (c_high-1)<<16, 256 entries.
 * intervals_dev must not be sym_dev or lut_dev; n above 2^31 - 1 CTAs of 256 is refused. */
int l3c_lut_intervals(const uint8_t *sym_dev, const uint32_t *lut_dev, int64_t n,
                      uint32_t *intervals_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * C. Discretised-logistic-mixture head
 *    (reference: criterion/logistic_mixture.py:134-275, torchac.py:174-213,
 *     torchac_kernel.cu:20-76, bitcoding.py:297-323)
 * ---------------------------------------------------------------------------------------- */

/* Shared CDF row of the uniform prior (bitcoding.py:297-323): L+1 uint16 entries written to
 * row_host (host-side helper, no device work). */
int l3c_uniform_cdf_row(int L, uint16_t *row_host);

/* Per-symbol coding intervals for all C channels of one scale of a batch.
 *   l_dev      f32 NHWC [N][HW][Kp], Kp = (rgb ? 4 : 3) * C * K, channel index p*C*K + c*K + k
 *   sym_dev    uint8 [N][C][HW]  symbols being coded (for RGB they are also the values that
 *              enter the mean coupling, logistic_mixture.py:262-272)
 *   targets_dev f32 [L+1] bin edges (coders_helpers.py:44-46)
 *   intervals_dev uint32 [N][C][HW] out */
int l3c_dmll_intervals(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev,
                       int N, int HW, int C, int K, int L, int rgb, uint32_t *intervals_dev,
                       void *stream);

/* uint16 CDF rows (pitch = 32 for L <= 32, else 256 entries) of channel c -- or of all C channels
 * when c < 0 (non-RGB scales: channels are conditionally independent) -- for pixels
 * [pix0, pix0+npix) of every image: table_dev[((n*C + c)*HW + p) * pitch + l].  For rgb && c > 0
 * the already decoded channels are read from sym_dev. */
int l3c_dmll_build_table(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev,
                         int N, int HW, int C, int K, int L, int rgb, int c, int pix0, int npix,
                         uint16_t *table_dev, int pitch, void *stream);

/* Tiled stream order (the codec's throughput mode): every H x W symbol plane is cut into tiles of th x tw
 * (smaller at the right / bottom edge), tiles in row-major tile order, symbols row-major inside a tile; each
 * tile is one coded stream.  l3c_dmll_build_table_tiled = l3c_dmll_build_table for ALL pixels with rows and
 * sym_dev indexed in tile order (l_dev stays raster NHWC).  l3c_reorder_tiles converts `planes` planes of
 * 1- or 4-byte elements between raster and tile order (to_tiles != 0: raster -> tiles); planes <= 65535 and
 * H * W < 2^31, else L3C_EINVAL.  A tile larger than the plane is the whole plane in that direction. */
int l3c_dmll_build_table_tiled(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev,
                               int N, int H, int W, int C, int K, int L, int rgb, int c, int th, int tw,
                               uint16_t *table_dev, int pitch, void *stream);
int l3c_reorder_tiles(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int H, int W, int th,
                      int tw, int to_tiles, void *stream);
/* Region decode (DESIGN §4.8): l3c_dmll_build_table_tiled for an H x W symbol plane whose parameters are the
 * rectangle at (oy, ox) of a wider plane, l_dev NHWC [N][Hl][Wl][Kp] (the output of a decoder window); rows and
 * sym_dev are in the tile order of the H x W plane.  Same rows as l3c_dmll_build_table_tiled on a copy of that
 * rectangle, without the copy.
 * l3c_crop_rect: the h x w rectangle at origins_dev[n] = (y, x) (int32 [N][2], inside the plane) of each of the
 * `planes` planes of image n: src N * planes planes of H x W elements of elem_bytes bytes -> dst N * planes planes
 * of h x w (NHWC tensors: planes = 1, elem_bytes = bytes per pixel). */
int l3c_dmll_build_table_window(const float *l_dev, int Hl, int Wl, int oy, int ox, const uint8_t *sym_dev,
                                const float *targets_dev, int N, int H, int W, int C, int K, int L, int rgb, int c,
                                int th, int tw, uint16_t *table_dev, int pitch, void *stream);
int l3c_crop_rect(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                  const int *origins_dev, int h, int w, void *stream);
/* One pass over region windows of different shapes (DESIGN §4.8 "Batches").
 * l3c_dmll_build_table_windows: l3c_dmll_build_table_window with a rectangle per image, geo_dev int32 [N][4] =
 * (oy, ox, H_n, W_n) (16-byte aligned): image n's rows and symbols are the tile order of its own H_n x W_n plane,
 * in stream-order planes of `plane` elements ((n * C + c) * plane), max_hw = max_n H_n * W_n.
 * l3c_crop_rects: l3c_crop_rect with a rectangle per image, rects_dev int32 [N][4] = (y, x, h_n, w_n) (16-byte
 * aligned).  dst_off_dev null: dst is N * planes planes of hp x wp, image n top-left and +0 elsewhere; otherwise image
 * n's planes of h_n x w_n follow each other from element dst_off_dev[n] (hp x wp: the largest rectangle); nothing
 * else of dst is written.  Every rectangle lies inside the H x W plane, and h_n <= hp, w_n <= wp.  Both crops refuse
 * a destination plane whose elements need more than 2^31 - 1 CTAs of 256 threads (bytes, or 4-byte words when
 * elem_bytes % 4 == 0).
 * l3c_reorder_tiles_images: uint8 tile order -> raster for images of different sizes: src N * planes planes of
 * plane_len bytes, image n's hold the tile order of its extents_dev[n] = (h_n, w_n) plane (int32 [N][2]); dst
 * N * planes planes of hp x wp, image n top-left and 0 elsewhere; h_n * w_n <= plane_len, and hp * wp < 2^31 (else
 * L3C_EINVAL). */
int l3c_dmll_build_table_windows(const float *l_dev, int Hl, int Wl, const int *geo_dev, int max_hw, int plane,
                                 const uint8_t *sym_dev, const float *targets_dev, int N, int C, int K, int L, int rgb,
                                 int c, int th, int tw, uint16_t *table_dev, int pitch, void *stream);
int l3c_crop_rects(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                   const int *rects_dev, const int64_t *dst_off_dev, int hp, int wp, void *stream);
int l3c_reorder_tiles_images(const uint8_t *src_dev, uint8_t *dst_dev, int planes, int N, int plane_len, int hp,
                             int wp, const int *extents_dev, int th, int tw, void *stream);

/* Negative log-likelihood (nats) summed per image: nll_dev f64 [N] (overwritten).
 * target value of symbol s is values_dev[s] (logistic_mixture.py:146-207). */
int l3c_dmll_nll(const float *l_dev, const uint8_t *sym_dev, const float *values_dev,
                 int N, int HW, int C, int K, int L, int rgb, float x_min, float x_max,
                 double *nll_dev, float *nll_map_dev /* f32 [N][C][HW] per-sub-pixel nats, or NULL */,
                 void *stream);

/* Reference-shaped per-channel mixture parameters (CDFOut, logistic_mixture.py:61-65,134-141,
 * 248-275): softmax(pi), mu (incl. RGB coupling from x_dec_dev f32 [N][C][HW]) and clamped
 * log sigma, each f32 [N][K][HW]. */
int l3c_dmll_channel_params(const float *l_dev, const float *x_dec_dev, int N, int HW, int C, int K,
                            int rgb, int c, float *pi_dev, float *mu_dev, float *log_scales_dev,
                            void *stream);

/* Sample every sub-pixel from its mixture (logistic_mixture.py:277-323; used by test.py --sample): Gumbel-max
 * choice of the component from u_sel_dev f32 [N][C][K][HW], inverse-CDF sample of its logistic from u_x_dev f32
 * [N][C][HW] (both uniform in [1e-5, 1 - 1e-5], supplied by the caller), RGB: means coupled through the
 * coefficients of the chosen components and values clamped to [0, 255].  x_dev f32 [N][C][HW] out. */
int l3c_dmll_sample(const float *l_dev, const float *u_sel_dev, const float *u_x_dev, int N, int HW, int C, int K,
                    int rgb, float *x_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * D. Convolution stack (reference: modules/net.py:89-184, edsr.py:52-119, head.py:26-59,
 *    prob_clf.py:29-74, pytorch_ext.py:57-61; all nn.Conv2d fp32)
 * ---------------------------------------------------------------------------------------- */

#define L3C_CONV_RELU 1u            /* y = max(y, 0) after bias                                  */
#define L3C_CONV_PIXEL_SHUFFLE2 2u  /* out[n,2h+i,2w+j,c] = y[n,h,w,4c+2i+j] (edsr.py:92-101)     */
#define L3C_CONV_ROUND_TF32 4u      /* (TF32 mode) round y itself to TF32 (cvt.rna): y only feeds tensor-core convs */

#define L3C_PREC_FP32 0             /* CUDA-core FFMA, fp32 throughout (bit-faithful ordering)    */
#define L3C_PREC_TF32 1             /* wgmma kind::tf32 on operands pre-rounded to TF32 (RN), fp32 accumulate in registers */
#define L3C_PREC_F16 2              /* wgmma kind::f16 on FP16 operand images (RN, saturating; the same 10 mantissa */
                                    /* bits as TF32-RN), fp32 accumulate in registers, fp32 residual stream               */
#define L3C_PREC_F16X2 3            /* strict tensor-core mode: every operand is the sum of two FP16 numbers, hi = fp16(x) */
                                    /* and lo = fp16((x - hi) * 2^11); a product is hi*hi + (hi*lo + lo*hi) / 2^11 = three   */
                                    /* wgmma into two register accumulators (the error-compensated split SURVEY section 7 */
                                    /* asks for, with FP16 instead of TF32 pieces): ~2^-22 relative, i.e. fp32-class results  */
                                    /* at several times the CUDA-core rate.  Operand images are [..][2*C] FP16: hi planes in  */
                                    /* channels [0,C), lo planes in [C,2C); 3x3/s1/Cin=64 and 1x1 layers                      */

typedef struct {
    const float *x;        /* dev NHWC [N][H][W][x_pitch] fp32, channels [0,Cin) read (FP32 / TF32 kernels)     */
    const float *w;        /* dev [KH][KW][Cin][cout_pad] (FP32) or the TF32 operand image (TF32)                */
    const float *bias;     /* dev [cout_pad]                                                       */
    const float *residual; /* dev NHWC like the output (same pitch/offset), or NULL: y += res      */
    float *y;              /* dev NHWC [N][Ho][Wo][y_pitch], channels [y_coff, y_coff+Cout) written; may be NULL  */
                           /* in F16 mode when only y_h is wanted                                                */
    float *y_tf32;         /* optional second output, same layout as y: the result rounded to TF32     */
                           /* (round-to-nearest) = operand image for a following TF32 tensor-core conv; NULL ok */
    void *y_h;             /* optional output, same element pitch/offset as y: the result as FP16 (RN, saturating) */
                           /* = operand image for a following F16 tensor-core conv; written by every kernel; NULL ok */
    const void *x_h;       /* F16 tensor-core kernels: FP16 operand image of the input, NHWC [N][H][W][x_pitch]    */
    const void *w_h;       /* F16 tensor-core kernels: FP16 weight image, 3x3: [9 taps][cout_pad][64],             */
                           /* 1x1: [Cin/64][cout_pad][64]                                                         */
    int N, H, W, Cin, x_pitch;
    int Cout, cout_pad, y_pitch, y_coff;
    int ksize, stride, dilation;   /* padding = ksize/2 if dilation==1 else dilation               */
    unsigned flags;
    int precision;
    int yh_pitch;          /* element pitch of y_h when it differs from y_pitch (0 = same): split images are 2x as wide */
    int yh_lo_off;         /* > 0: y_h is a SPLIT image (L3C_PREC_F16X2): lo plane yh_lo_off elements after the hi plane */
} l3c_conv_t;

int l3c_conv2d(const l3c_conv_t *p, void *stream);

/* The DMLL head fused into the 1x1 `lin` conv of the probability classifier (encode side; reference:
 * prob_clf.py:71-74 followed by logistic_mixture.py:248-275 and torchac_kernel.cu:26-76): the Kp parameters of
 * a pixel never reach HBM -- the conv's epilogue evaluates the two CDF bounds of every coded symbol directly
 * from the accumulator.  x_h: FP16 operand image NHWC [N][HW][Cin] (the atrous concat); w_h: FP16 weight image
 * [Cin/64][cout_pad][64]; bias f32 [cout_pad]; sym_dev uint8 [N][C][HW]; targets_dev f32 [L+1];
 * intervals_dev uint32 [N][C][HW] out, bit-identical to l3c_conv2d (F16) + l3c_dmll_intervals. */
int l3c_lin_dmll_intervals(const void *x_h, const void *w_h, const float *bias, const uint8_t *sym_dev,
                           const float *targets_dev, int N, int HW, int Cin, int C, int K, int L, int rgb,
                           uint32_t *intervals_dev, void *stream);

/* The intervals of one band of a banded encode in f16 (DESIGN §4.10): as l3c_lin_dmll_intervals on rows [oy, oy + h)
 * of x_h, the FP16 concat buffer [N][Hl][W][Cin] of a full-width decoder window, coding the symbols of rows
 * [y0, y0 + h) of the whole symbol plane sym_dev uint8 [N][C][Hs][W]; their intervals written in the tile order
 * (th x tw) of an h x W plane to band stream planes intervals_dev uint32 [N][C][h * W].  Bit-identical to the
 * whole-plane kernel followed by l3c_reorder_tiles, restricted to the band. */
int l3c_lin_dmll_intervals_band(const void *x_h, int Hl, int oy, const void *w_h, const float *bias,
                                const uint8_t *sym_dev, int Hs, int y0, int h, int W, const float *targets_dev, int N,
                                int Cin, int C, int K, int L, int rgb, int th, int tw, uint32_t *intervals_dev,
                                void *stream);

/* The intervals of one tile-aligned rectangle of a banded encode (a band: x0 = 0, w = Ws of a whole plane) or of a
 * region update (DESIGN §4.10, §4.12): as l3c_dmll_intervals for the h x w rectangle at (y0, x0) of the symbol window
 * sym_dev uint8 [N][C][Hs][Ws], which sits at (sy, sx) of the container's Hf x Wf plane, with the parameters at
 * (oy, ox) of l_dev f32 NHWC [N][Hl][Wl][Kp]; intervals in the tile order (th x tw) of an h x w plane to
 * intervals_dev uint32 [N][C][h * w].  In the Hf x Wf plane the rectangle starts on a tile boundary and ends on one
 * or at the plane's edge (else an error), so its tile order is that of the plane's own tiles.  Bit-identical to the
 * whole-plane kernel followed by l3c_reorder_tiles, restricted to the rectangle. */
int l3c_dmll_intervals_rect(const float *l_dev, int Hl, int Wl, int oy, int ox, const uint8_t *sym_dev, int Hs, int Ws,
                            int y0, int x0, int h, int w, int sy, int sx, int Hf, int Wf, const float *targets_dev,
                            int N, int C, int K, int L, int rgb, int th, int tw, uint32_t *intervals_dev,
                            void *stream);
/* l3c_dmll_intervals_rect with one rectangle per image, for a pass of region updates whose windows differ in shape
 * (DESIGN §4.12, "Batches of updates"): geo_host int32 [N][10] = (oy, ox, y0, x0, h_n, w_n, sy, sx, Hf, Wf) per image:
 * the rectangle's origin in image n's parameters (l_dev f32 NHWC [N][Hl][Wl][Kp], a padded batch of decoder outputs),
 * its origin and size in image n's symbol window (sym_dev uint8 [N][C][Hs][Ws], a padded batch), that window's origin
 * in image n's Hf x Wf plane and the plane's size.  Image n's intervals go, in the tile order (th x tw, shared) of its
 * own h_n x w_n rectangle, to its stream planes intervals_dev uint32 [N][C][plane] from element (n * C + c) * plane;
 * nothing past h_n * w_n of a plane is written.  The geometry is copied to geo_dev (device, 4-byte aligned, N * 40 bytes)
 * on `stream` before the launch.  Refused before any GPU work (L3C_EINVAL), for any image: what l3c_dmll_intervals_rect
 * refuses (a rectangle outside the parameters, the symbol window or the plane, or not tile-aligned in the plane; C, K,
 * L; null pointers), and h_n * w_n > plane.  Bit-identical to l3c_dmll_intervals_rect run on every image alone. */
int l3c_dmll_intervals_rects(const float *l_dev, int Hl, int Wl, const uint8_t *sym_dev, int Hs, int Ws,
                             const int *geo_host, int *geo_dev, int plane, const float *targets_dev, int N, int C, int K,
                             int L, int rgb, int th, int tw, uint32_t *intervals_dev, void *stream);

/* sub_rgb_mean + first MeanShift of RGBHead as one per-pixel 3x3 affine pair
 * (multiscale_network.py:181-183, head.py:31-33): img uint8 [N][3][HW] planes ->
 * x_sub f32 NHWC [N][HW][3] (= A1 img + b1)  and  t f32 NHWC [N][HW][4] (= A2 x_sub + b2, ch 3 = 0).
 * A1,b1,A2,b2: dev f32 [9],[3],[9],[3] (the two 1x1 conv parameter sets). Either output may be NULL. */
int l3c_rgb_prep(const uint8_t *img_dev, const float *A1, const float *b1, const float *A2,
                 const float *b2, int N, int HW, float *xsub_dev, float *t_dev, void *stream);

/* F16 path of the RGB head (head.py:26-59): the two MeanShift affines of l3c_rgb_prep followed by an im2col of the
 * 3x3 neighbourhood: out_h_dev FP16 [N][HW][64], element (ky*3+kx)*3 + c = normalised channel c at tap (ky,kx)
 * (0 outside the image), elements 27..63 zero -- the 3 -> 64 conv then runs as a K = 64 GEMM on the tensor cores. */
int l3c_rgb_im2col_f16(const uint8_t *img_dev, const float *A1, const float *b1, const float *A2, const float *b2,
                       int N, int H, int W, void *out_h_dev, void *stream);
/* l3c_rgb_im2col_f16 for a ragged batch (DESIGN §4.6): image n occupies [0,h_n) x [0,w_n) of the padded H x W
 * planes, extents_dev int32 [N][2] = (h_n, w_n), and taps outside that extent are 0 as at the tensor border.
 * extents_dev = NULL is l3c_rgb_im2col_f16. */
int l3c_rgb_im2col_f16_ragged(const uint8_t *img_dev, const float *A1, const float *b1, const float *A2,
                              const float *b2, int N, int H, int W, const int *extents_dev, void *out_h_dev,
                              void *stream);

/* Ragged batches (DESIGN §4.6): padded NHWC / planar tensors in which image n occupies [0,h_n) x [0,w_n);
 * extents_dev int32 [N][2] = (h_n, w_n) at the tensor's resolution.
 * l3c_ragged_zero_halo: sets the band of `halo` pixels right of and below every image, [h_n, h_n + halo) x
 * [0, w_n + halo) and [0, h_n) x [w_n, w_n + halo) clipped to the tensor, of an NHWC tensor with px_bytes bytes per
 * pixel (a multiple of 4) to +0, and nothing else -- run on the input of a k x k conv, it gives every output pixel
 * inside its image the operands of the per-image launch.
 * l3c_ragged_pack: N * planes planes of H x W elements of elem_bytes bytes (plane n * planes + q belongs to image
 * n); to_compact != 0: padded raster -> compact planes of compact_len elements holding the h_n * w_n elements of
 * the image row-major, then zeros; to_compact == 0: compact -> padded raster with zeros outside the image.  Every
 * extent lies inside H x W and h_n * w_n <= compact_len.  Both refuse a plane (compact_len or H * W elements) that
 * needs more than 2^31 - 1 CTAs of 256 threads. */
int l3c_ragged_zero_halo(void *x_dev, int px_bytes, int N, int H, int W, const int *extents_dev, int halo,
                         void *stream);
int l3c_ragged_pack(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                    const int *extents_dev, long long compact_len, int to_compact, void *stream);
/* l3c_dmll_nll of a ragged batch: l_dev NHWC [N][H][W][Kp] and sym_dev [N][C][H][W] are padded, nll_dev f64 [N]
 * gets the nats of the h_n * w_n pixels of every image, bit-identical to l3c_dmll_nll on that image alone (the same
 * 128-pixel blocks in raster order of the extent, the same summation order).  Nothing outside an extent is read.
 * Every extent must satisfy 1 <= h_n <= H and 1 <= w_n <= W; an image whose extent does not reads nothing and
 * gets NaN. */
int l3c_dmll_nll_ragged(const float *l_dev, const uint8_t *sym_dev, const float *values_dev, int N, int H, int W,
                        int C, int K, int L, int rgb, float x_min, float x_max, const int *extents_dev,
                        double *nll_dev, void *stream);

/* L3C_PREC_F16X2: fp32 [n_px][C] -> split operand image FP16 [n_px][2*C] (hi = fp16(x) in channels [0,C),
 * lo = fp16((x - hi) * 2^11) in [C,2C)); C % 4 == 0.  For the outputs of the CUDA-core layers of that mode (no
 * reference counterpart: the reference's convolutions are cuDNN fp32, pytorch_models/modules/edsr.py:33-38). */
int l3c_split_f16x2(const float *x_dev, long long n_px, int C, void *out_h_dev, void *stream);

/* to_q 1x1 conv + hard quantiser (net.py:116-148, quantizer.py:62-90):
 * sym = argmin_l (q - level_l)^2 (first minimum), bn_q = levels[sym].
 * f_dev NHWC [N][HW][Cf]; w_dev [Cf][C]; bias [C]; levels [L];
 * sym_dev uint8 [N][C][HW] planes; bnq_dev f32 NHWC [N][HW][C]. */
int l3c_quantize_head(const float *f_dev, const float *w_dev, const float *bias_dev,
                      const float *levels_dev, int N, int HW, int Cf, int C, int L,
                      uint8_t *sym_dev, float *bnq_dev, void *stream);

/* bn = values[sym] for symbol planes -> NHWC f32 [N][HW][C] minus optional per-channel shift
 * (decode side of quantizer.py:44-47 / SURVEY finding 1, and the RGB baselines' x - rgb_mean). */
int l3c_symbols_to_values(const uint8_t *sym_dev, const float *values_dev, const float *shift_dev,
                          int N, int HW, int C, int L, float *out_dev, void *stream);

/* Pillow-compatible bicubic x0.5 on uint8 planes [N][3][H][W] -> [N][3][H/2][W/2]
 * (dataloaders/images_loader.py:277-293 via PIL.Image.resize(BICUBIC); RGB baselines only). */
int l3c_bicubic_half_u8(const uint8_t *in_dev, int N, int H, int W, uint8_t *out_dev, void *stream);

/* RGB scale of a decode, channel-pipelined, as ONE host call (the runtime loop of codec.py moved into the
 * library: ~400 launches and event operations per decode): chunk j of channel c-1 decoded -> rows of chunk j of
 * channel c built on bld_streams[c] -> channel c's decoders resume on dec_streams[c] (state carried in the
 * descriptors).  desc_dev_per_channel[c]: device array of N stream descriptors of channel c.  Ordered after
 * `cur_stream`'s queue; `cur_stream` waits for all of it.  Reference: the strictly serial R -> G -> B loop of
 * bitcoding.py:199-237. */
int l3c_decode_rgb_pipelined(const float *l_dev, uint8_t *sym_dev, const float *targets_dev, int N, int HW, int K,
                             int L, uint16_t *table_dev, int pitch,
                             const l3c_dec_stream_t *const *desc_dev_per_channel, int chunk_px, void *cur_stream,
                             void *const *bld_streams, void *const *dec_streams, int coarse);
/* coarse != 0: table_dev holds coarse records instead of rows (pitch = 96, see l3c_dmll_build_coarse), built by
 * l3c_dmll_build_coarse and decoded by l3c_ac_decode_streams_coarse; same symbols, same saved states. */

/* Coarse CDF rows of RGB channel c (L = 256, K = 10) for pixels [pix0, pix0+npix) of every image: per sub-pixel one
 * record of 96 uint16 at rec_dev[((n*3 + c)*HW + p) * 96]: the channel's mixture parameters as 32 floats (pi[10],
 * mu[10], -log2(e)/sigma[10], 2 zeros), then the 32 entries cdf[8 i], i = 0..31, of the full row that
 * l3c_dmll_build_table builds (cdf[256] = 2^16 is implied).  sym_dev: the decoded R (and G) symbols for c > 0. */
int l3c_dmll_build_coarse(const float *l_dev, const uint8_t *sym_dev, const float *targets_dev, int N, int HW, int K,
                          int L, int c, int pix0, int npix, uint16_t *rec_dev, void *stream);
/* l3c_dmll_build_coarse on decoder windows (region decodes of seek-indexed reference-layout containers, DESIGN §4.13
 * "Regions"): image n's parameters are the rectangle geo_dev[n] = (oy, ox, H_n, W_n) (int32 [N][4], 16-byte aligned)
 * of l_dev NHWC [N][Hl][Wl][120]; its records and decoded symbols are in the raster order of that H_n x W_n rectangle,
 * in planes of `plane` elements (record of sub-pixel p of channel c at rec_dev[((n*3 + c)*plane + p) * 96]),
 * max_hw = max_n H_n * W_n.  Null pointers, L != 256, c outside 0..2, c > 0 without sym_dev and max_hw outside
 * 1..plane are refused (L3C_EINVAL) before anything is launched. */
int l3c_dmll_build_coarse_windows(const float *l_dev, int Hl, int Wl, const int *geo_dev, int max_hw, int plane,
                                  const uint8_t *sym_dev, const float *targets_dev, int N, int K, int L, int c,
                                  uint16_t *rec_dev, void *stream);
/* l3c_ac_decode_streams for L = 256 with every stream's `table` pointing at coarse records (row_pitch >= 96, 4-byte
 * aligned); targets_dev: the 256 bin targets the records were built with.  The entries between two coarse entries
 * are evaluated on demand, with the builder's arithmetic: symbols and saved states equal a full-row decode. */
int l3c_ac_decode_streams_coarse(const l3c_dec_stream_t *streams_dev, int n_streams, const float *targets_dev,
                                 uint32_t first, uint32_t count, void *stream);

/* ------------------------------------------------------------------------------------------
 * F. torchac, batched: the drop-in's streams, many per launch (l3c_pytorch_b200.torchac.*_batch)
 *    Section A codes one stream per synchronous call.  These two kernels turn the sources of any number of streams
 *    into the inputs of section B's coder: coding intervals for l3c_ac_encode_streams, decoder rows for
 *    l3c_ac_decode_streams.  The integers are those of section A for the same stream.  The host composes them:
 *    one interval launch, one encode launch and one pack for a whole call; the rows chunk by chunk, the decoder
 *    resuming from its saved state.  Asynchronous on `stream`; nothing is allocated.
 * ---------------------------------------------------------------------------------------- */

/* The source of one stream.  A table stream has `table` set; a mixture stream has table = NULL and the four
 * plane pointers set.  Lp = L + 1 as in section A (2 to 32769, checked by the caller).  The kernels assume valid
 * descriptors and do not check them. */
typedef struct {
    const uint16_t *table;      /* dev [n_sym][Lp]: the 1HWLp CDF tensor, flattened; or NULL                      */
    const float *targets;       /* mixture: dev f32 [Lp]                                                            */
    const float *means;         /* mixture: dev f32 [K][n_sym]                                                      */
    const float *log_scales;    /* mixture: dev f32 [K][n_sym] (unclamped, as in l3c_encode_logistic_mixture)      */
    const float *probs;         /* mixture: dev f32 [K][n_sym]                                                      */
    const int16_t *sym;         /* dev int16 [n_sym]: the symbols to code (read by l3c_batch_intervals only)       */
    int64_t n_sym;              /* 1 to 2^31 - 1                                                                    */
    int32_t Lp;
    int32_t K;                  /* mixture components (>= 1); ignored for a table stream                            */
} l3c_code_src_t;

/* Coding intervals of every symbol of every stream, one launch.  sym_off_dev int64 [n_streams + 1]: prefix sums of
 * n_sym (sym_off[0] = 0, sym_off[n_streams] = n_total); stream j's intervals go to intervals_dev + sym_off[j], packed
 * c_low | (c_high - 1) << 16 as table_intervals_kernel / plane_intervals_kernel (section A) produce them.
 * bad_dev int32 [n_streams]: stream j's first position whose symbol lies outside [0, Lp - 2], or -1 if there is
 * none; such a symbol's interval is written as 0 and nothing else is read for it. */
int l3c_batch_intervals(const l3c_code_src_t *src_dev, const int64_t *sym_off_dev, int n_streams, int64_t n_total,
                        uint32_t *intervals_dev, int32_t *bad_dev, void *stream);

/* Decoder rows of symbols [first, first + r_j) of every stream j, r_j = min(count, n_sym - first) (0 if
 * first >= n_sym), one launch.  row_off_dev int64 [n_streams + 1], in uint16 entries: stream j's rows start at
 * rows_dev + row_off[j], and row_off[j + 1] - row_off[j] = r_j * pitch_j with pitch_j the decoder's pitch for
 * L = Lp - 1 (32 for L <= 32, 256 for L <= 256, else round_up(L, 8)); n_entries = row_off[n_streams].  rows_dev
 * must be 16-byte aligned.  Entries 0..L-1 of a row are the CDF (a table row, or the mixture row that
 * l3c_decode_logistic_mixture builds), the rest are 0.  A descriptor of l3c_ac_decode_streams then points its
 * `table` at rows_dev + row_off[j] - first * pitch_j, so that symbol first + i reads row i. */
int l3c_batch_rows(const l3c_code_src_t *src_dev, const int64_t *row_off_dev, int n_streams, int64_t n_entries,
                   uint32_t first, uint16_t *rows_dev, void *stream);

/* ------------------------------------------------------------------------------------------
 * E. Execution resources
 * ---------------------------------------------------------------------------------------- */

/* Streams confined to two disjoint groups of SMs of the current device (driver green contexts):
 * `n_a` streams (high priority) whose kernels only run on a group of about `sm_a` SMs (the driver
 * rounds up to its granularity, 8 on sm_90+), `n_b` streams on the remaining SMs (all but the last of
 * them high priority, the last one default priority).  Used by the
 * pipelined RGB decode (reference: the strictly serial R -> G -> B loop of bitcoding.py:199-237) so
 * that the latency-bound decoder warps do not share SMs with the CDF-row builders.  The streams
 * belong to the primary context (same memory, events interoperate) and live until process exit;
 * repeated calls with the same `sm_a` return the same streams.  *sm_a_out / *sm_b_out (optional)
 * receive the actual group sizes.  L3C_EUNSUPPORTED if the driver cannot partition: the caller then
 * uses ordinary streams (slower, same results). */
int l3c_partition_streams(int sm_a, int n_a, void **streams_a, int n_b, void **streams_b,
                          int *sm_a_out, int *sm_b_out);
/* the same with explicit counts of high- and default-priority streams on the remaining SMs */
int l3c_partition_streams2(int sm_a, int n_a, void **streams_a, int n_b_high, void **streams_b_high,
                           int n_b_low, void **streams_b_low, int *sm_a_out, int *sm_b_out);

/* Test knob for the persistent tensor-core convolutions (3x3, 5x5/s2, 1x1, fused DMLL head), process-wide, from
 * the next launch on.  0 = default for either argument.
 *   max_sms > 0:      the SM count these kernels size their grid with becomes min(max_sms, SMs of the stream's
 *                     partition group or of the device) -- few CTAs, many tiles per CTA and per pipe.
 *   conv_smem_kb > 0: replaces L3C_CONV_SMEM_KB as the shared-memory budget (KB, clamped to [112, 227]) from which
 *                     the FP16 kernels choose their number of pipeline stages.
 * Lets small inputs exercise the stage rings, both pipes and every stage count; with both at 0 every launch
 * configuration is the default one.  Not meant for production use. */
int l3c_set_conv_launch_limits(int max_sms, int conv_smem_kb);

/* Test and diagnosis knob for the persistent tensor-core convolutions, process-wide, from the next launch on: how
 * a launch hands its tiles to its CTAs.
 *   0: dynamic (default): each pipe claims its next tile from a per-launch counter, so CTAs that start late run
 *      fewer tiles;
 *   1: static stripe: CTA b runs tiles b, b + G, ... (G = gridDim.x), its two pipes alternating;
 *   2: dynamic with a start skew: odd CTAs wait 500 us before their first claim, so a few CTAs take most tiles
 *      and some take none.
 * Every mode gives the same bits.  Any other value is L3C_EINVAL.  Not meant for production use. */
int l3c_set_conv_tile_schedule(int mode);

/* *count = CTAs of the current device that ran no tile under schedule mode 2 since the last reset (waits for the
 * device); reset != 0 then zeroes the count.  Not meant for production use. */
int l3c_conv_idle_ctas(long long *count, int reset);

/* One CTA of a persistent tensor-core convolution, as a library built with L3C_CTA_TRACE records it
 * (`python -m l3c_pytorch_b200.build --cta-trace`, tools/cta_timeline.py). */
typedef struct {
    uint64_t t_start;   /* %globaltimer (ns) at the CTA's first instruction */
    uint64_t t_end;     /* %globaltimer when the CTA's last warp left */
    uint32_t smid;      /* the SM it ran on */
    uint32_t tiles;     /* the tiles its consumers ran */
    uint32_t launch;    /* launch index since l3c_cta_trace_register */
    uint32_t cta;       /* blockIdx.y * gridDim.x + blockIdx.x */
} l3c_cta_record_t;

/* L3C_CTA_TRACE builds: from the next launch on, the CTAs of every persistent tensor-core launch write their
 * records into records_dev (device memory, `capacity` records; launches that do not fit any more are not recorded)
 * and the launch index starts from 0.  records_dev = NULL stops the recording.  Other builds: L3C_EUNSUPPORTED. */
int l3c_cta_trace_register(l3c_cta_record_t *records_dev, int64_t capacity);
/* L3C_CTA_TRACE builds: one line "launch name grid_x grid_y first_record stream" per launch since the last
 * l3c_cta_trace_register (truncated to `cap`); *n_records = records written.  Other builds: L3C_EUNSUPPORTED. */
int l3c_cta_trace_launches(char *buf, size_t cap, int64_t *n_records);

/* Test knob for the range decoder of alphabets L > 32, process-wide, from the next launch on: streams per CTA (1, 2
 * or 4) of v3::ac_decode_kernel<FULLROW, SPC>; 0 = the L3C_DEC_SPC environment variable or, without it, the default
 * (2).  Any other value is L3C_EINVAL.  Lets one process run every variant, including a partial last CTA.  Not meant
 * for production use. */
int l3c_set_decoder_streams_per_cta(int spc);

/* Test knob: streams per CTA (1, 2 or 4) of ac_encode_kernel<SPC>, each stream a coding warp and an emitter warp;
 * 0 = the L3C_ENC_SPC environment variable or, without it, the default (4).  Any other value is L3C_EINVAL.  Lets
 * one process run every variant, including a partial last CTA.  Not meant for production use. */
int l3c_set_encoder_streams_per_cta(int spc);

/* Test probe of the CDF rows' sigmoid: for the n fp32 values u_dev[i] (device), raw_dev[i] = sigmoid_from_log2(u)
 * (~ 1 / (1 + 2^u), the MUFU.EX2 + MUFU.RCP evaluation every CDF entry uses) and term_dev[i] = mixture_term(0, 1, u)
 * (the same with the saturation shortcuts: exactly 1 for u <= -25, 0 for u >= 40).  Both call the kernels' own
 * __device__ functions, so a test can measure what the built library computes.  Not meant for production use. */
int l3c_dmll_probe_sigmoid(const float *u_dev, float *raw_dev, float *term_dev, int64_t n, void *stream);

/* ------------------------------------------------------------------------------------------
 * G. Training (l3c_pytorch_b200.train; reference: criterion/logistic_mixture.py:146-207,
 *    modules/quantizer.py:62-90): the two per-pixel losses of a training step, forward and
 *    backward, on the NCHW fp32 tensors nn.Conv2d produces.  A NULL gradient pointer selects the
 *    forward.  The backward reads the upstream gradient from device memory (no host sync) and
 *    recomputes everything from the forward's inputs; every gradient element is written once, so
 *    results are bit-identical from run to run.
 * ---------------------------------------------------------------------------------------- */

/* DMLL negative log-likelihood of one scale, as train.dmll_nll computes it.
 *   l_dev  f32 [N][Kp][HW], Kp = (rgb ? 4 : 3) * C * K, channel p*C*K + c*K + k (p: 0 logits, 1 means,
 *          2 log-scales, 3 RGB coefficients); K = 10
 *   x_dev  f32 [N][C][HW] targets (RGB: the pixel values; bottleneck: the soft quantiser's values)
 *   half_bin, x_lower, x_upper: half the bin width and the edge-branch thresholds (x < x_lower: lower branch,
 *          x > x_upper: upper branch), as fp32.
 * Forward (grad_dev NULL): nll_dev f64 [N] = the nats of every image, summed per 128 pixels and then per image in a
 * fixed order (two launches).  Backward: grad_dev f32 [1] the upstream gradient of the summed nats; dl_dev f32 like
 * l_dev, every plane written; dx_dev f32 like x_dev or NULL (must be NULL when rgb).  One launch. */
int l3c_dmll_nll_train(const float *l_dev, const float *x_dev, int N, int HW, int C, int K, int rgb, float half_bin,
                       float x_lower, float x_upper, double *nll_dev, const float *grad_dev, float *dl_dev,
                       float *dx_dev, void *stream);

/* Soft quantiser of n fp32 values q_dev onto levels_dev f32 [L] (1 <= L <= 256).
 * Forward (grad_dev NULL): sym_dev int64 [n] = the first l minimising (q - level_l)^2, value_dev f32 [n] =
 * levels[sym].  Backward: dq_dev f32 [n] = grad_dev[i] * 2 sigma Var_phi(levels), phi = softmax_l(-sigma (q -
 * level_l)^2) (sigma > 0): the gradient of the soft value sum_l level_l phi_l that the hard value stands in for. */
int l3c_soft_quantize(const float *q_dev, int64_t n, const float *levels_dev, int L, float sigma, int64_t *sym_dev,
                      float *value_dev, const float *grad_dev, float *dq_dev, void *stream);

/* Backward of the 3x3, stride-1, 64-input-channel convolutions (padding = dilation = d in {1, 2, 4}, Cout in {64,
 * 256}) on the TF32 tensor cores, fp32 accumulation.  Tensors are NHWC fp32: x [N][H][W][64], dy [N][H][W][Cout],
 * dx [N][H][W][64].  Every call checks its arguments before any GPU work and refuses (L3C_EINVAL) null pointers,
 * Cin != 64, Cout not in {64, 256}, d not in {1, 2, 4}, N not in [1, 65535], H * W above 2^30 (MAX_PLANE_PIXELS)
 * and pointers that are not 16-byte aligned (so an element offset that is not a multiple of 64 bits is refused).
 * Every output element is written once, in a fixed order: the same inputs give the same bits on every run. */

/* y_dev[i] = x_dev[i] rounded to TF32 (cvt.rna), n values; y_dev may be x_dev.  The operand image the TF32 kernels
 * read (the tensor cores would otherwise truncate). */
int l3c_round_tf32(const float *x_dev, float *y_dev, int64_t n, void *stream);

/* Data gradient: dx = the 3x3 conv of dy with the weights flipped spatially and Cin / Cout swapped, no bias, run by
 * the forward TF32 kernel (conv3x3_tf32_kernel).  dy_dev must hold TF32-rounded values (l3c_round_tf32).
 * w_dev: the flipped image [Cout / 64][9 taps][2 K-halves][64 ci][32 co] fp32, TF32-rounded; slice s reads the
 * channels 64s..64s+63 of dy, and the Cout / 64 slices are added in order 0, 1, ... through the kernel's residual
 * epilogue (Cout / 64 launches). */
int l3c_conv3x3_dgrad(const float *dy_dev, const float *w_dev, int N, int H, int W, int Cin, int Cout, int dilation,
                      float *dx_dev, void *stream);

/* Bytes of the workspace l3c_conv3x3_wgrad needs for this shape (0 for an invalid one). */
int64_t l3c_conv3x3_wgrad_workspace(int N, int H, int W, int Cout);

/* Weight and bias gradient: dw_dev [Cout][64][3][3] (OIHW, as nn.Conv2d's weight) = sum over n, y, x of
 * dy[n, y, x, co] * x[n, y + d (ky - 1), x + d (kx - 1), ci] (x = 0 outside the image); db_dev [Cout] = sum of dy.
 * The pixels are split into chunks of whole 8x16 tiles, one chunk per CTA (the split depends on the shape only);
 * each CTA accumulates its chunk with mma.sync m16n8k8 TF32 on operands rounded to TF32 (RN) and writes its partial
 * sums to work_dev, then a second launch adds the chunks in chunk order.  No atomics. */
int l3c_conv3x3_wgrad(const float *x_dev, const float *dy_dev, int N, int H, int W, int Cin, int Cout, int dilation,
                      float *dw_dev, float *db_dev, float *work_dev, int64_t work_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* L3C_B200_H_ */
