// xray_pyramid.cuh — kernels of the X-ray pipeline beyond the leaf tile (SURVEY 8 f3): binned columns, the background
// pass, parent tiles (2 x 2 mosaic + Lanczos3 reduction).  The per-element arithmetic lives in xray_pyramid.h (shared with the
// sequential test backend); the kernels here only distribute elements over threads.
// All of it is HBM-bound byte work: one coalesced read and one coalesced write of every image per pass; a parent tile of
// 4096^2 pixels reads 4 x 64 MB of children and writes 128 MB + 64 MB.
#pragma once
#include "query.cuh"
#include "xray_pyramid.h"

namespace pcv {

// assign_background (xray/src/generation.rs:695-720) in place.
__global__ void __launch_bounds__(256) k_xray_background(uint32_t* __restrict__ rgba, size_t npix, uint32_t bg) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) rgba[i] = background_pixel(rgba[i], bg);
}

// vertical_sample over the (virtual) mosaic: out is [out_h][in_w] RGBA; consecutive threads take consecutive columns.
struct ResampleVArgs {
    MosaicSrc src;
    ResampleTaps taps;
    uint32_t in_w, out_h;
    uint32_t* out;
};
__global__ void __launch_bounds__(256) k_xray_resample_v(const __grid_constant__ ResampleVArgs a) {
    const size_t n = (size_t)a.in_w * a.out_h;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t oy = (uint32_t)(i / a.in_w), x = (uint32_t)(i % a.in_w);
        a.out[i] = resample_v_pixel(a.src, a.taps, x, oy);
    }
}
// horizontal_sample: in is [h][in_w], out is [h][out_w].
struct ResampleHArgs {
    const uint32_t* in;
    ResampleTaps taps;
    uint32_t in_w, out_w, h;
    uint32_t* out;
};
__global__ void __launch_bounds__(256) k_xray_resample_h(const __grid_constant__ ResampleHArgs a) {
    const size_t n = (size_t)a.out_w * a.h;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / a.out_w), ox = (uint32_t)(i % a.out_w);
        a.out[i] = resample_h_pixel(a.in + (size_t)y * a.in_w, a.taps, ox);
    }
}

// ---- binned columns: PointColor (MODE 1) / Intensity (MODE 2) strategies with Binning = Some(("intensity", size)) --------
__global__ void __launch_bounds__(256) k_fill_u64(uint64_t* __restrict__ dst, uint64_t value, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = value;
}
struct XrayBinnedArgs {
    XrayArgs x;
    const uint8_t* rgb;      // node-contiguous colours
    const float* intensity;  // node-contiguous intensities (the binning attribute; the value in mode 2)
    double bin_size;
    BinnedTables t;
};
// Per point: the pixel of k_xray_accum_attr (xray_pixel), then the (pixel, bin) hash aggregation of xray_pyramid.h.
template <int MODE>
__global__ void __launch_bounds__(256) k_xray_binned_insert(const __grid_constant__ XrayBinnedArgs b) {
    const XrayArgs& a = b.x;
    const QTile t = a.tiles[blockIdx.x];
    const QNode nd = a.nodes[t.node];
    const int bpc = enc_bytes(nd.enc);
    bool seen = false;
    for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
        double p[3];
        decode_point(a.xyz, nd, bpc, t.first + i, p);
        if (!loc_contains(a.geom, p[0], p[1], p[2])) continue;
        seen = true;
        uint32_t x, y, z;
        xray_pixel(a, p, x, y, z);
        if (!(x < a.w && y < a.h)) continue;
        const uint32_t px = y * a.w + x;
        const uint64_t slot = nd.point_off + t.first + i;
        const float inten = b.intensity[slot];
        const int64_t bin = xray_bin_of(inten, b.bin_size);
        float v[3];
        if (MODE == 1) {  // Color<u8>::to_f32: f32::from(c) / 255.
            const uint8_t* c = b.rgb + 3 * slot;
            v[0] = (float)c[0] / 255.f, v[1] = (float)c[1] / 255.f, v[2] = (float)c[2] / 255.f;
        } else {
            if (inten < 0.f) continue;
            v[0] = inten;
        }
        binned_insert(b.t, px, bin, v);
    }
    if (__syncthreads_or(seen) && threadIdx.x == 0) atomicExch(a.any, 1);
}
__global__ void __launch_bounds__(256) k_xray_binned_reduce(const BinnedTables t, float* __restrict__ pix_sum, int stride, uint32_t* __restrict__ pix_bins) {
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < t.col_cap; s += (uint64_t)gridDim.x * blockDim.x)
        binned_reduce_slot(t, s, pix_sum, stride, pix_bins);
}

}  // namespace pcv
