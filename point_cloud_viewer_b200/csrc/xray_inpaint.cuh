// xray_inpaint.cuh — kernels of inpaint_xray_quadtree (xray/src/inpaint.rs) over one block of leaves (xray_inpaint.inl):
// every leaf of the block's 1-halo gets a 2T x 2T inpaint image stitched from the visible tiles of its 3 x 3 neighbourhood,
// closed, filled from its nearest sample, blended with its Right and Bottom neighbours' images, and cropped.
// Images are RGBA packed in a u32 (r | g << 8 | b << 16 | a << 24), row-major, row 0 at the top (the tile's PNG row order);
// spatial y grows upwards, so the Top neighbour (y + 1) lies above.  Every pass is exact integer or IEEE f32 arithmetic; the
// line passes take one thread per image row or column and cost O(2T) per line whatever the inpaint distance.
#pragma once
#include "xray_pyramid.cuh"

namespace pcv {

constexpr uint32_t kInpaintTransparent = 0x00FFFFFFu;  // TRANSPARENT.to_u8() (src/color.rs:154): the stitched image's empty pixels

struct InpaintArgs {
    const uint32_t* tiles;    // [tile slot][T * T]
    const int32_t* tile_slot; // [(B + 4)^2] tile grid, row-major, row 0 at the top: slot or -1
    const uint32_t* pos;      // [image] ix | iy << 16 in the (B + 2)^2 image grid (image (ix, iy) = tile (ix + 1, iy + 1))
    uint32_t* img;            // [image][2T * 2T]
    uint8_t* m1;              // [image][2T * 2T] masks
    uint8_t* m2;
    int32_t* near_row;        // [image][2T * 2T] column pass: the nearest sample's row in this column, or -1
    int32_t* env;             // [image][2T * 2T] row pass: the lower envelope's columns, per row
    unsigned long long* holes;  // [image] hole pixels
    uint32_t T, G, nimg, k;     // tile edge, tile grid edge (B + 4), images, inpaint distance
};

// stitched_image (inpaint.rs:90-121): the 2T x 2T window of the plane of tiles centred on the leaf; the copy_subimage regions of
// the 8 neighbours are exactly the window's pixels that fall into them.
__global__ void __launch_bounds__(256) k_inpaint_stitch(const __grid_constant__ InpaintArgs a) {
    const uint32_t S = 2 * a.T, w = a.T / 2;
    const size_t n = (size_t)a.nimg * S * S;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t im = (uint32_t)(i / ((size_t)S * S)), p = (uint32_t)(i % ((size_t)S * S));
        const int du = (int)(p % S) - (int)w, dv = (int)(p / S) - (int)w;
        const int dx = du < 0 ? -1 : (du >= (int)a.T ? 1 : 0), dy = dv < 0 ? -1 : (dv >= (int)a.T ? 1 : 0);
        const uint32_t gx = (a.pos[im] & 0xFFFFu) + 1 + dx, gy = (a.pos[im] >> 16) + 1 + dy;
        const int32_t slot = a.tile_slot[gy * a.G + gx];
        a.img[i] = slot < 0 ? kInpaintTransparent
                            : a.tiles[(size_t)slot * a.T * a.T + (size_t)(dv - dy * (int)a.T) * a.T + (uint32_t)(du - dx * (int)a.T)];
    }
}

// One pass of close(mask, LInf, k) (imageproc morphology): per line, a running count of the set source pixels in the window
// [p - k, p + k] clipped to the image.  MODE 0: source alpha != 0, out = any set (dilation, rows); 1: source m, any set
// (dilation, columns); 2: source m, all set (erosion, rows); 3: all set (erosion, columns), then out = closed and alpha == 0
// (the pixels to fill), counted per image.  ROWS: one thread per row, else one per column.
template <bool ROWS, int MODE>
__global__ void __launch_bounds__(128) k_inpaint_window(const __grid_constant__ InpaintArgs a, const uint8_t* __restrict__ src, uint8_t* __restrict__ out) {
    const uint32_t S = 2 * a.T, line = blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= a.nimg * S) return;
    const uint32_t im = line / S, l = line % S;
    const size_t base = (size_t)im * S * S + (ROWS ? (size_t)l * S : l), step = ROWS ? 1 : S;
    auto set = [&](uint32_t p) -> uint32_t { return MODE == 0 ? (a.img[base + p * step] >> 24 != 0u) : (uint32_t)src[base + p * step]; };
    const int k = (int)a.k, n = (int)S;
    uint32_t cnt = 0;
    for (int p = 0; p <= k && p < n; ++p) cnt += set(p);
    unsigned long long holes = 0;
    for (int p = 0; p < n; ++p) {
        const uint32_t len = (uint32_t)(min(p + k, n - 1) - max(p - k, 0) + 1);
        uint8_t v = MODE <= 1 ? (cnt != 0) : (cnt == len);
        if (MODE == 3) {
            v = v && (a.img[base + (size_t)p * step] >> 24) == 0u;
            holes += v;
        }
        out[base + (size_t)p * step] = v;
        if (p + k + 1 < n) cnt += set(p + k + 1);
        if (p - k >= 0) cnt -= set(p - k);
    }
    if (MODE == 3 && holes) atomicAdd(&a.holes[im], holes);
}

// The column pass of the nearest-sample transform: per pixel, the row of the nearest sample (alpha != 0) in its column, the
// upper one on a tie; -1 when the column holds none.  One thread per column.
__global__ void __launch_bounds__(128) k_inpaint_near_col(const __grid_constant__ InpaintArgs a) {
    const uint32_t S = 2 * a.T, line = blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= a.nimg * S) return;
    const size_t base = (size_t)(line / S) * S * S + line % S;
    int last = -1;  // downwards: the nearest sample at or above
    for (uint32_t r = 0; r < S; ++r) {
        if (a.img[base + (size_t)r * S] >> 24) last = (int)r;
        a.near_row[base + (size_t)r * S] = last;
    }
    int next = -1;  // upwards: the nearest sample at or below; the upper one wins a tie
    for (int r = (int)S - 1; r >= 0; --r) {
        if (a.img[base + (size_t)r * S] >> 24) next = r;
        const int up = a.near_row[base + (size_t)r * S];
        if (next >= 0 && (up < 0 || next - r < r - up)) a.near_row[base + (size_t)r * S] = next;
    }
}

// The row pass (lower envelope of the parabolas (c - q)^2 + (r - near_row[q])^2 over the columns q that hold a sample), then
// the fill: every hole pixel of the row (m2) takes the pixel of its nearest sample, the smaller column on a tie.  Holes are
// never samples, so the rows read by one thread are never written by another.  One thread per row; rows without a hole skip.
__global__ void __launch_bounds__(128) k_inpaint_fill_row(const __grid_constant__ InpaintArgs a) {
    const uint32_t S = 2 * a.T, line = blockIdx.x * blockDim.x + threadIdx.x;
    if (line >= a.nimg * S) return;
    const size_t base = (size_t)(line / S) * S * S + (size_t)(line % S) * S;
    const int64_t r = line % S;
    const uint8_t* hole = a.m2 + base;
    bool any = false;
    for (uint32_t c = 0; c < S && !any; ++c) any = hole[c] != 0;
    if (!any) return;
    const int32_t* nr = a.near_row + base;
    int32_t* v = a.env + base;
    auto f = [&](int64_t q) { const int64_t d = r - nr[q]; return d * d; };
    // the envelope's parabolas by column; z[k] = crossing of v[k - 1] and v[k] = num / den, compared exactly
    int top = -1;
    for (int64_t q = 0; q < S; ++q) {
        if (nr[q] < 0) continue;
        while (top >= 1) {
            const int64_t p = v[top], o = v[top - 1];
            const int64_t n1 = (f(p) + p * p) - (f(o) + o * o), d1 = 2 * (p - o);  // z[top]
            const int64_t n2 = (f(q) + q * q) - (f(p) + p * p), d2 = 2 * (q - p);  // crossing of v[top] and q
            if (n2 * d1 <= n1 * d2) --top;
            else break;
        }
        v[++top] = (int32_t)q;
    }
    int kk = 0;
    for (int64_t c = 0; c < S; ++c) {
        if (!hole[c]) continue;
        auto val = [&](int64_t q) { return (c - q) * (c - q) + f(q); };
        while (kk < top && val(v[kk + 1]) < val(v[kk])) ++kk;
        const int64_t q = v[kk];
        a.img[base + c] = a.img[(size_t)(line / S) * S * S + (size_t)nr[q] * S + q];
    }
}

// interpolate_subimages (utils.rs:47-83): value = (n * wt + c * (1 - wt)).round() per channel, written into both images.
__device__ __forceinline__ uint32_t inpaint_blend(uint32_t n, uint32_t c, float wt) {
    const float wc = __fsub_rn(1.0f, wt);
    uint32_t out = 0;
    for (int s = 0; s < 32; s += 8) {
        const float v = __fadd_rn(__fmul_rn((float)((n >> s) & 255u), wt), __fmul_rn((float)((c >> s) & 255u), wc));
        out |= (uint32_t)img_f32_to_u8(v) << s;
    }
    return out;
}
// interpolate_inpaint_image_with (inpaint.rs:132-161): pair (current, neighbour).  VERTICAL false: Right, current columns
// [T, 2T) with the neighbour's [0, T), the neighbour weighted i / (T - 1) by column; true: Bottom, the same on rows.
template <bool VERTICAL>
__global__ void __launch_bounds__(256) k_inpaint_blend(const __grid_constant__ InpaintArgs a, const int2* __restrict__ pairs, uint32_t npairs) {
    const uint32_t S = 2 * a.T;
    const size_t half = (size_t)a.T * S, n = (size_t)npairs * half;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int2 pr = pairs[i / half];
        const uint32_t e = (uint32_t)(i % half);
        uint32_t row, col, t;  // t: the position along the blend (the weight's i or j)
        if (VERTICAL) row = e / S, col = e % S, t = row;
        else row = e / a.T, col = e % a.T, t = col;
        const float wt = __fdiv_rn((float)t, (float)(a.T - 1));
        uint32_t* cur = a.img + (size_t)pr.x * S * S + (VERTICAL ? (size_t)(row + a.T) * S + col : (size_t)row * S + col + a.T);
        uint32_t* nb = a.img + (size_t)pr.y * S * S + (size_t)row * S + col;
        const uint32_t v = inpaint_blend(*nb, *cur, wt);
        *cur = v;
        *nb = v;
    }
}

// apply_inpainting (inpaint.rs:163-173): the centre T x T of image `im`, then assign_background_color's alpha < 128 rule.
__global__ void __launch_bounds__(256) k_inpaint_crop(const __grid_constant__ InpaintArgs a, uint32_t im, uint32_t bg, uint32_t* __restrict__ out) {
    const uint32_t S = 2 * a.T, w = a.T / 2;
    const size_t n = (size_t)a.T * a.T;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(i / a.T), c = (uint32_t)(i % a.T);
        out[i] = background_pixel(a.img[(size_t)im * S * S + (size_t)(r + w) * S + c + w], bg);
    }
}

}  // namespace pcv
