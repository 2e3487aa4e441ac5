// ragged.cu -- batches of differently sized images (DESIGN §4.6).
//
// A ragged batch is a padded batch [N][Hmax][Wmax][..] in which image n occupies [0,h_n) x [0,w_n) at the
// finest scale and (h_n >> s, w_n >> s) at scale s.  `extents_dev` is int32 [N][2] = (h_n, w_n) at the
// resolution of the tensor a call works on.
//   * l3c_ragged_zero_halo: the margin band [h_n, h_n + halo) x [0, w_n + halo) and [0, h_n) x [w_n, w_n + halo)
//     of every image (clipped to the tensor) is set to +0.  Run on the input of a k x k conv before it is launched,
//     it makes every operand an output pixel inside its image reads equal to what the per-image launch reads
//     (there the zeros come from TMA's out-of-bounds fill), so the bits are identical.
//   * l3c_ragged_pack: padded raster planes <-> per-image compact planes ("stream order" of the range coder:
//     plane q of image n holds its h_n * w_n elements row-major at [(n * planes + q) * compact_len], the tail up
//     to compact_len is zero).  Gathers intervals and mixture parameters for the coder, scatters decoded symbols
//     back into zero-padded planes.
#include "common.cuh"

namespace l3c {

__global__ void zero_halo_kernel(uint32_t *__restrict__ x, int words_per_px, int H, int W,
                                 const int *__restrict__ ext, int halo) {
    const int n = blockIdx.y;
    const int h = min(ext[2 * n], H), w = min(ext[2 * n + 1], W);
    const int wr = (int)min((int64_t)w + halo, (int64_t)W), hb = (int)min((int64_t)h + halo, (int64_t)H);
    const int64_t right = (int64_t)h * (wr - w);                 // [0,h) x [w,wr)
    const int64_t count = right + (int64_t)(hb - h) * wr;         // + [h,hb) x [0,wr)
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t px = r / words_per_px;
    if (px >= count) return;
    int y, xx;
    if (px < right) {
        y = (int)(px / (wr - w));
        xx = w + (int)(px % (wr - w));
    } else {
        const int64_t j = px - right;
        y = h + (int)(j / wr);
        xx = (int)(j % wr);
    }
    x[(((int64_t)n * H + y) * W + xx) * words_per_px + r % words_per_px] = 0u;
}

template <typename T>
__global__ void ragged_pack_kernel(const T *__restrict__ src, T *__restrict__ dst, int per_elem, int planes, int H,
                                   int W, const int *__restrict__ ext, int64_t compact_len, int to_compact) {
    const int plane = blockIdx.y;
    const int n = plane / planes;
    const int h = ext[2 * n], w = ext[2 * n + 1];
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t e = r / per_elem, k = r % per_elem;
    const int64_t padded = (int64_t)plane * H * W, compact = (int64_t)plane * compact_len;
    if (to_compact) {
        if (e >= compact_len) return;
        T v = 0;
        if (e < (int64_t)h * w) {
            const int64_t y = e / w, x = e % w;
            v = src[(padded + y * W + x) * per_elem + k];
        }
        dst[(compact + e) * per_elem + k] = v;
    } else {
        if (e >= (int64_t)H * W) return;
        const int64_t y = e / W, x = e % W;
        T v = 0;
        if (y < h && x < w) v = src[(compact + y * w + x) * per_elem + k];
        dst[(padded + e) * per_elem + k] = v;
    }
}

}  // namespace l3c

extern "C" int l3c_ragged_zero_halo(void *x_dev, int px_bytes, int N, int H, int W, const int *extents_dev, int halo,
                                    void *stream) {
    using namespace l3c;
    L3C_REQUIRE(x_dev && extents_dev, "l3c_ragged_zero_halo: null pointer");
    L3C_REQUIRE(px_bytes >= 4 && px_bytes % 4 == 0 && N >= 1 && N <= 65535 && H >= 1 && W >= 1 && halo >= 0,
                "l3c_ragged_zero_halo: px_bytes=%d N=%d H=%d W=%d halo=%d", px_bytes, N, H, W, halo);
    if (halo == 0) return L3C_OK;
    const int wpp = px_bytes / 4;
    halo = halo < (H > W ? H : W) ? halo : (H > W ? H : W);      // a wider band is clipped to the same pixels
    const int64_t band = (int64_t)halo * ((int64_t)H + W);       // bound on the band of any image, in pixels
    L3C_REQUIRE(fits_grid_x(band, wpp), "l3c_ragged_zero_halo: a %d-pixel band of %dx%d pixels of %d bytes", halo, H, W,
                px_bytes);
    dim3 grid((unsigned)ceil_div64(band * wpp, 256), N);
    zero_halo_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint32_t *)x_dev, wpp, H, W, extents_dev, halo);
    L3C_LAUNCH_CHECK("zero_halo_kernel");
    return L3C_OK;
}

extern "C" int l3c_ragged_pack(const void *src_dev, void *dst_dev, int elem_bytes, int planes, int N, int H, int W,
                               const int *extents_dev, long long compact_len, int to_compact, void *stream) {
    using namespace l3c;
    L3C_REQUIRE(src_dev && dst_dev && src_dev != dst_dev && extents_dev, "l3c_ragged_pack: bad pointers");
    L3C_REQUIRE(elem_bytes >= 1 && planes >= 1 && N >= 1 && (int64_t)N * planes <= 65535 && H >= 1 && W >= 1 &&
                    compact_len >= 1,
                "l3c_ragged_pack: elem_bytes=%d planes=%d N=%d H=%d W=%d compact_len=%lld", elem_bytes, planes, N, H, W,
                compact_len);
    const bool words = elem_bytes % 4 == 0;
    const int per_elem = words ? elem_bytes / 4 : elem_bytes;
    const int64_t len = to_compact ? (int64_t)compact_len : (int64_t)H * W;
    L3C_REQUIRE(fits_grid_x(len, per_elem), "l3c_ragged_pack: planes of %lld elements of %d bytes in one launch",
                (long long)len, elem_bytes);
    dim3 grid((unsigned)ceil_div64(len * per_elem, 256), N * planes);
    if (words)
        ragged_pack_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint32_t *)src_dev, (uint32_t *)dst_dev, per_elem, planes, H, W, extents_dev, compact_len, to_compact);
    else
        ragged_pack_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>(
            (const uint8_t *)src_dev, (uint8_t *)dst_dev, per_elem, planes, H, W, extents_dev, compact_len, to_compact);
    L3C_LAUNCH_CHECK("ragged_pack_kernel");
    return L3C_OK;
}
