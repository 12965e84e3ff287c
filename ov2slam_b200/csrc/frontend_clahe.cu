// C: contrast-limited adaptive histogram equalisation (cv::CLAHE semantics), bit-exact.
//
// Reference behaviour replaced: pclahe_->apply(img, img) with cv::createCLAHE(fclahe_val = 3,
// Size(W/50, H/50)) (/root/reference/src/ov2slam.cpp:85-89, applied at src/visual_front_end.cpp:
// 1158-1160 and src/mapper.cpp:75-76; `use_clahe: 1`, i.e. the accurate/ configurations).
// Algorithm (SURVEY.md A.6, pinned against cv2 by oracle/image_ref.py::clahe_ref):
//   * if W % tx or H % ty != 0 the image is extended right by tx - W % tx AND bottom by ty - H % ty
//     (both, REFLECT_101); tile = extended size / tiles
//   * per tile 256-bin histogram, clip = max(int(clip * area / 256), 1), excess redistributed
//     (uniform batch + one each to bins 0, step, 2 step, ...), LUT = rint(cumsum * (255 / area))
//   * per pixel float32 bilinear blend of the four neighbouring tile LUTs, rint.
// clahe_lut_kernel: one warp per (tile, frame), one shared-memory histogram per warp from 32-bit loads.
// clahe_apply_kernel: one CTA per (band of rows between two tile-centre lines, frame), its two LUT rows staged in
// shared memory, streaming pass with 32-bit loads / stores (reads W*H, writes W*H per frame).
#include "ov2_common.cuh"

namespace {

struct ClaheArgs {
    const uint8_t* src; uint8_t* dst;
    int w, h, spitch, dpitch;
    long long sfstride, dfstride;
    int tx, ty, tw, th, clip;
    float lut_scale, inv_tw, inv_th;
    uint8_t* lut;   // [count][ty][tx][256]
};

__device__ __forceinline__ int refl(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i;
}

// Tile histogram -> clipped, redistributed -> LUT.  One WARP per (tile, frame), eight tiles per CTA, no block barrier:
// with 52 x 52-pixel tiles (1280 x 720, 25 x 14 tiles) a CTA per tile spent more instructions zeroing, merging and
// scanning eight sub-histograms (and waiting at five barriers) than counting.  A warp keeps ONE 256-bin histogram in shared
// memory, counts 4 pixels per 32-bit load (interior tiles whose rows are 4-byte addressable; tiles that reach into the
// reflected extension, or unaligned images, take the byte path), then every lane owns 8 consecutive bins for the clip,
// the redistribution (uniform batch + one each to bins 0, step, 2 step, ...) and the prefix sum (8 local + one warp scan).
constexpr int LUT_WARPS = 8;
__global__ void __launch_bounds__(LUT_WARPS * 32) clahe_lut_kernel(ClaheArgs A) {
    __shared__ __align__(16) int whist[LUT_WARPS][256];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x * LUT_WARPS + warp, fr = blockIdx.y;
    if (tile >= A.tx * A.ty) return;
    const int tyi = tile / A.tx, txi = tile - tyi * A.tx;
    const uint8_t* src = A.src + A.sfstride * fr;
    int* hist = whist[warp];
#pragma unroll
    for (int k = 0; k < 8; ++k) hist[lane + 32 * k] = 0;
    __syncwarp();
    const int x0 = txi * A.tw, y0 = tyi * A.th;
    const bool words = x0 + A.tw <= A.w && y0 + A.th <= A.h && (A.tw & 3) == 0 && (x0 & 3) == 0 && (A.spitch & 3) == 0 &&
                       ((reinterpret_cast<uintptr_t>(src)) & 3) == 0;
    if (words) {
        const int wpr = A.tw >> 2, nw = wpr * A.th;
        const int dy = 32 / wpr, dx = 32 - dy * wpr;
        int yy = lane / wpr, xw = lane - yy * wpr;
        const uint32_t* base = reinterpret_cast<const uint32_t*>(src + (size_t)y0 * A.spitch + x0);
        const int wpitch = A.spitch >> 2;
        for (int i = lane; i < nw; i += 128) {               // four loads in flight per lane
            uint32_t v[4];
            bool ok[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                ok[u] = i + 32 * u < nw;
                v[u] = ok[u] ? __ldg(base + (size_t)yy * wpitch + xw) : 0u;
                xw += dx; yy += dy;
                if (xw >= wpr) { xw -= wpr; yy++; }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (ok[u]) {
                    atomicAdd(&hist[v[u] & 255u], 1);
                    atomicAdd(&hist[(v[u] >> 8) & 255u], 1);
                    atomicAdd(&hist[(v[u] >> 16) & 255u], 1);
                    atomicAdd(&hist[v[u] >> 24], 1);
                }
        }
    } else {
        const int area = A.tw * A.th;
        const int dy = 32 / A.tw, dx = 32 - dy * A.tw;
        int yy = lane / A.tw, xx = lane - yy * A.tw;
        for (int i = lane; i < area; i += 32) {
            const int x = refl(x0 + xx, A.w), y = refl(y0 + yy, A.h);
            atomicAdd(&hist[__ldg(src + (size_t)y * A.spitch + x)], 1);
            xx += dx; yy += dy;
            if (xx >= A.tw) { xx -= A.tw; yy++; }
        }
    }
    __syncwarp();
    // lane owns bins 8 lane .. 8 lane + 7
    int v[8];
    {
        const int4 a = *reinterpret_cast<const int4*>(hist + 8 * lane), b = *reinterpret_cast<const int4*>(hist + 8 * lane + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    int excess = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (v[k] > A.clip) { excess += v[k] - A.clip; v[k] = A.clip; }
    const int clipped = __reduce_add_sync(0xffffffffu, excess);
    const int batch = clipped >> 8;
    const int residual = clipped - (batch << 8);
    if (residual != 0) {
        const int step = max(256 / residual, 1);
        const unsigned inv = (65536u + (unsigned)step - 1u) / (unsigned)step;    // floor(b / step) = (b inv) >> 16 for b < 256, step <= 256
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const unsigned b = 8u * lane + k, q = (b * inv) >> 16;
            // bins 0, step, 2*step, ... (the first `residual` of them, while index < 256)
            if (b - q * step == 0u && (int)q < residual) v[k]++;
        }
    }
    int sum = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { v[k] += batch; sum += v[k]; v[k] = sum; }      // local inclusive prefix
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    const int basec = incl - sum;
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int q = __float2int_rn((float)(basec + v[k]) * A.lut_scale);
        q = q < 0 ? 0 : (q > 255 ? 255 : q);
        if (k < 4) lo |= (uint32_t)q << (8 * k);
        else hi |= (uint32_t)q << (8 * (k - 4));
    }
    uint8_t* out = A.lut + (((size_t)fr * A.ty + tyi) * A.tx + txi) * 256 + 8 * lane;
    *reinterpret_cast<uint2*>(out) = make_uint2(lo, hi);
}

// Interpolation pass.  All rows between two tile-centre lines use the same two LUT rows (ty1, ty2): one CTA takes such a
// band of one frame, stages those two LUT rows (2 x tiles_x x 256 bytes) in shared memory with coalesced loads, then
// streams the band: 4 pixels per thread and step (one 32-bit load, one 32-bit store), the four LUT gathers per pixel hit
// shared memory instead of L1/L2.  Reads W*H, writes W*H per frame.
constexpr int APPLY_MAX_TX = 64;
__global__ void __launch_bounds__(512) clahe_apply_kernel(ClaheArgs A) {
    extern __shared__ uint8_t s_lut[];                       // [2][tx][256]
    const int fr = blockIdx.y, band = blockIdx.x;            // band b: rows whose floor(y / th - 0.5) == b - 1
    const uint8_t* lut = A.lut + (size_t)fr * A.ty * A.tx * 256;
    // rows of this band: ty1 = b - 1 (clamped), ty2 = b (clamped)
    int ylo = 0, yhi = A.h;
    {
        // tyf = y * inv_th - 0.5 in float, floor -> band index - 1; find the row range by scanning the candidates around
        // the analytic boundary (th / 2 + (b - 1) * th) so the float rounding of the kernel's own expression decides
        const int c0 = (band - 1) * A.th + A.th / 2;
        ylo = max(0, c0 - 2); yhi = min(A.h, c0 + A.th + 2);
    }
    const int t1 = max(band - 1, 0), t2 = min(band, A.ty - 1);
    const int lut_row = A.tx * 256;
    for (int i = threadIdx.x * 16; i < lut_row; i += blockDim.x * 16) {
        *reinterpret_cast<uint4*>(s_lut + i) = __ldg(reinterpret_cast<const uint4*>(lut + (size_t)t1 * lut_row + i));
        *reinterpret_cast<uint4*>(s_lut + lut_row + i) = __ldg(reinterpret_cast<const uint4*>(lut + (size_t)t2 * lut_row + i));
    }
    __syncthreads();
    const uint8_t* l1 = s_lut;
    const uint8_t* l2 = s_lut + lut_row;
    const bool words = ((A.spitch | A.dpitch) & 3) == 0 && ((reinterpret_cast<uintptr_t>(A.src + A.sfstride * fr) | reinterpret_cast<uintptr_t>(A.dst + A.dfstride * fr)) & 3) == 0;
    const int wq = (A.w + 3) >> 2;
    // first / last row of the band by the kernel's own float expression (candidates around the analytic boundary)
    int ya_ = yhi, yb_ = ylo;
    for (int y = ylo; y < yhi; ++y)
        if (__float2int_rd((float)y * A.inv_th - 0.5f) == band - 1) { ya_ = min(ya_, y); yb_ = max(yb_, y + 1); }
    // column-stationary: a thread keeps the horizontal interpolation data of its 4 pixels (two LUT column offsets and the
    // two weights each - they depend on x only) in registers and walks down the rows of the band
    for (int xw = threadIdx.x; xw < wq; xw += blockDim.x) {
        const int xq = xw * 4;
        int o1[4], o2[4];
        float wa[4], wb[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float txf = (float)(xq + k) * A.inv_tw - 0.5f;
            int tx1 = __float2int_rd(txf);
            wa[k] = txf - (float)tx1;
            wb[k] = 1.0f - wa[k];
            int tx2 = tx1 + 1;
            tx1 = max(tx1, 0);
            tx2 = min(tx2, A.tx - 1);
            o1[k] = tx1 * 256; o2[k] = tx2 * 256;
        }
        const bool full = words && xq + 4 <= A.w;
        for (int y = ya_; y < yb_; ++y) {
            const float tyf = (float)y * A.inv_th - 0.5f;
            const float ya = tyf - (float)(band - 1), ya1 = 1.0f - ya;
            const uint8_t* srow = A.src + A.sfstride * fr + (size_t)y * A.spitch;
            uint8_t* drow = A.dst + A.dfstride * fr + (size_t)y * A.dpitch;
            uint32_t in;
            if (full) in = __ldg(reinterpret_cast<const uint32_t*>(srow + xq));
            else { in = 0; for (int k = 0; k < 4 && xq + k < A.w; ++k) in |= (uint32_t)srow[xq + k] << (8 * k); }
            uint32_t out = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int v = (in >> (8 * k)) & 255;
                // byte -> float and float -> nearest int WITHOUT the conversion unit (I2F / F2I issue at a quarter of the
                // FP32 rate; five of them per pixel): 2^23 + b is exactly the float with mantissa b, and r + 1.5 * 2^23
                // rounds r to nearest-even into the mantissa - the same values as (float)b and rint(r).  0.68 -> 0.65 ms per
                // C4 step; staging the LUT rows as floats instead (4x the shared memory) measured slower, 0.71 ms.
                const float a11 = __uint_as_float(0x4B000000u | l1[o1[k] + v]) - 8388608.0f;
                const float a12 = __uint_as_float(0x4B000000u | l1[o2[k] + v]) - 8388608.0f;
                const float a21 = __uint_as_float(0x4B000000u | l2[o1[k] + v]) - 8388608.0f;
                const float a22 = __uint_as_float(0x4B000000u | l2[o2[k] + v]) - 8388608.0f;
                const float r = (a11 * wb[k] + a12 * wa[k]) * ya1 + (a21 * wb[k] + a22 * wa[k]) * ya;
                int q = __float_as_int(r + 12582912.0f) - 0x4B400000;
                q = q < 0 ? 0 : (q > 255 ? 255 : q);
                out |= (uint32_t)q << (8 * k);
            }
            if (full) *reinterpret_cast<uint32_t*>(drow + xq) = out;
            else for (int k = 0; k < 4 && xq + k < A.w; ++k) drow[xq + k] = (uint8_t)(out >> (8 * k));
        }
    }
}

}  // namespace

// shared by ov2_clahe and ov2_preprocess: everything on the device already
static ov2_status clahe_device(ov2_ctx* ctx, const uint8_t* src, int spitch, long long sfstride, uint8_t* dst, int dpitch,
                               long long dfstride, int width, int height, int count, double clip_limit, int tiles_x, int tiles_y) {
    ClaheArgs A;
    A.src = src; A.dst = dst;
    A.w = width; A.h = height; A.spitch = spitch; A.dpitch = dpitch;
    A.sfstride = sfstride; A.dfstride = dfstride;
    A.tx = tiles_x; A.ty = tiles_y;
    int ew = width, eh = height;
    if (width % tiles_x != 0 || height % tiles_y != 0) {      // OpenCV extends BOTH dimensions
        ew = width + (tiles_x - width % tiles_x);
        eh = height + (tiles_y - height % tiles_y);
    }
    A.tw = ew / tiles_x; A.th = eh / tiles_y;
    const int area = A.tw * A.th;
    int clip = 0;
    if (clip_limit > 0.0) {
        clip = (int)(clip_limit * area / 256);
        if (clip < 1) clip = 1;
    } else {
        clip = 1 << 30;
    }
    A.clip = clip;
    A.lut_scale = (float)255 / (float)area;
    A.inv_tw = 1.0f / (float)A.tw;
    A.inv_th = 1.0f / (float)A.th;
    ov2_status st;
    if ((st = ov2_scratch(ctx, (size_t)count * tiles_x * tiles_y * 256, A.lut)) != OV2_OK) return st;
    OV2_LAUNCH(ctx, "clahe_lut_kernel", clahe_lut_kernel<<<dim3((tiles_x * tiles_y + LUT_WARPS - 1) / LUT_WARPS, count), LUT_WARPS * 32, 0, ctx->stream>>>(A));
    if (tiles_x > APPLY_MAX_TX) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_clahe: more than 64 tile columns");
    {
        const size_t smem = (size_t)2 * tiles_x * 256;
        if (smem > 48 * 1024) OV2_CUDA(ctx, cudaFuncSetAttribute(clahe_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        // bands 0 .. tiles_y: rows above the first / below the last tile-centre line clamp to one LUT row
        int nthr = ((((width + 3) >> 2) + 31) / 32) * 32;                  // one thread per 4-pixel column of the image
        if (nthr > 512) nthr = 512;
        OV2_LAUNCH(ctx, "clahe_apply_kernel", clahe_apply_kernel<<<dim3(tiles_y + 1, count), nthr, smem, ctx->stream>>>(A));
    }
    return OV2_OK;
}

extern "C" ov2_status ov2_clahe(ov2_ctx* ctx, const uint8_t* src, uint8_t* dst, int width, int height, size_t row_stride,
                                size_t frame_stride, int count, double clip_limit, int tiles_x, int tiles_y) {
    if (!ctx || !src || !dst || width <= 0 || height <= 0 || count <= 0 || tiles_x <= 0 || tiles_y <= 0 ||
        row_stride < (size_t)width)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_clahe: bad arguments");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    const size_t bytes = frame_stride * (size_t)(count - 1) + row_stride * (size_t)(height - 1) + (size_t)width;
    const uint8_t* d = nullptr;
    uint8_t* o = nullptr;
    if ((st = ov2_stage_in(ctx, src, bytes, d)) != OV2_OK) return st;
    // a host dst is copied back over the whole span: when rows or frames leave gaps (a ROI of a wider image), stage its
    // current bytes first so the gaps come back unchanged
    const bool gaps = row_stride != (size_t)width || (count > 1 && frame_stride != row_stride * (size_t)height);
    if ((st = ov2_stage_out(ctx, dst, bytes, o, gaps)) != OV2_OK) return st;
    if ((st = clahe_device(ctx, d, (int)row_stride, (long long)frame_stride, o, (int)row_stride,
                           (long long)frame_stride, width, height, count, clip_limit, tiles_x, tiles_y)) != OV2_OK)
        return st;
    return ov2_end(ctx);
}

// VisualFrontEnd::preprocessImage (/root/reference/src/visual_front_end.cpp:1143-1177; the right image:
// src/mapper.cpp:75-81): optional CLAHE of the raw image, then buildOpticalFlowPyramid.  `raw` keeps the
// untouched image (describeBRIEF reads it, src/map_manager.cpp:301-303,326-329), `out` receives the
// equalised level 0 in its own storage and levels 1.. built from it: the image crosses PCIe once.
extern "C" ov2_status ov2_preprocess(ov2_ctx* ctx, const ov2_pyr* raw, ov2_pyr* out, int first, int count, int use_clahe,
                                     double clip_limit, int tiles_x, int tiles_y) {
    if (!ctx || !raw || !out || first < 0 || count <= 0 || first + count > raw->batch || first + count > out->batch ||
        raw->w[0] != out->w[0] || raw->h[0] != out->h[0] || !raw->l0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_preprocess: bad arguments / raw pyramid not loaded");
    if (use_clahe && (tiles_x <= 0 || tiles_y <= 0)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_preprocess: bad tile grid");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    if (!use_clahe) {
        // no equalisation: the tracking image IS the raw image -> alias it
        if (out->l0_mode == 1) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_preprocess: output pyramid owns level 0");
        out->l0 = raw->l0; out->l0_pitch = raw->l0_pitch; out->l0_fstride = raw->l0_fstride; out->l0_mode = 2;
    } else {
        if (out->l0_mode == 2) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_preprocess: output pyramid aliases device images");
        if (!out->own[0]) {
            OV2_CUDA(ctx, cudaMalloc(&out->own[0], out->fstride[0] * (size_t)out->batch));
            out->l0 = out->own[0]; out->l0_pitch = out->pitch[0]; out->l0_fstride = out->fstride[0]; out->l0_mode = 1;
        }
        if ((st = clahe_device(ctx, raw->l0 + raw->l0_fstride * (size_t)first, (int)raw->l0_pitch, (long long)raw->l0_fstride,
                               out->own[0] + out->fstride[0] * (size_t)first, (int)out->pitch[0], (long long)out->fstride[0],
                               raw->w[0], raw->h[0], count, clip_limit, tiles_x, tiles_y)) != OV2_OK)
            return st;
    }
    if ((st = ov2_pyr_make_levels(ctx, out, first, count)) != OV2_OK) return st;
    return ov2_end(ctx);
}
