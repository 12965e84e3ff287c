// R: rectification / undistortion (cv::remap, INTER_LINEAR, BORDER_CONSTANT 0, 8-bit, one channel), bit-exact.
//
// Reference behaviour replaced: CameraCalibration::rectifyImage (/root/reference/src/camera_calibration.cpp:233-241),
// cv::remap(img, rect, undist_map_x_, undist_map_y_, cv::INTER_LINEAR), run on every incoming image when `bdo_stereo_rect`
// or `bdo_undist` is set (src/ov2slam.cpp:239-243, 252-257).  Its maps come from setUndistStereoMap (CV_16SC2 + CV_16UC1,
// :141) or setUndistMap (CV_32FC1 x / y, :92); fisheye maps are the same data.
//
// Both map types reduce to one per-pixel entry (built once, by remap_convert_kernel):
//   CV_16SC2 + CV_16UC1: (X, Y) = map1, a = map2 & 31, b = (map2 >> 5) & 31
//   CV_32FC1:            X32 = rint(x * 32) (half to even; out of int range: a miss), X = X32 >> 5, a = X32 & 31, same for y
//                        - what cv::convertMaps(.., CV_16SC2) computes, and cv::remap with float maps equals that path.
// Packed entry (uint32): bits 0-10 X + 1, 11-21 Y + 1, 22-26 a, 27-31 b; REMAP_MISS when the 2 x 2 footprint lies wholly
// outside the image.  X + 1 <= W <= 2046 for every footprint that touches the image, so 2047 is free for the miss code.
// Per pixel, with p = 0 outside the image (BORDER_CONSTANT, value 0):
//   s = (32-a)(32-b) p(Y,X) + a(32-b) p(Y,X+1) + (32-a)b p(Y+1,X) + ab p(Y+1,X+1)
//   out = (32 s + 2^14) >> 15 = (s + 512) >> 10            (<= 255: the weights sum to 1024, no clamp needed)
// pinned against cv2.remap by oracle/remap_ref.py.
//
// remap_kernel: 256 threads, a CTA owns a 128 x 8 tile of the map (4 horizontally adjacent entries per thread, one 16-byte
// load, kept in registers) and applies it to every frame of its frame group: per frame and pixel 4 byte gathers and one
// byte of a 32-bit store.  Designed to be HBM-bound: about 1 B read (the source footprint of a tile is a slightly warped
// tile, its lines are shared by neighbouring pixels and rows) and 1 B written per pixel, the map's 4 B per pixel paid once
// per frame group.  The gathers go through L1 (__ldg); staging the footprint's bounding box in shared memory was not built.
// Measured (H100 80GB HBM3 SXM, 400 W limit, 132 frames of 752 x 480, scripts/bench_rect.py): 0.155 ms per launch, 626 GB/s of
// algorithmic bytes, 19 % of the 3.35 TB/s data-sheet bandwidth - the four byte gathers per pixel through L1 bound it, not HBM.
// 64 registers (launch bound: 4 CTAs per SM), no shared memory.  Frame groups (grid.z) exist only to fill the SMs when an
// image has few tiles; a batch of 752 x 480 images (360 tiles) uses 3.
#include "ov2_common.cuh"

struct ov2_remap_map {
    int device = 0;
    int w = 0, h = 0;
    int pitch = 0;            // entries per row (multiple of 4; padding entries are REMAP_MISS)
    uint32_t* entries = nullptr;
};

namespace {

constexpr uint32_t REMAP_MISS = 0xFFFFFFFFu;
constexpr int RT_X = 32, RT_Y = 8;          // threads
constexpr int R_TILE_W = 4 * RT_X;          // 128 map entries per tile row
constexpr int REMAP_MAX_SIDE = 2046;

__device__ __forceinline__ uint32_t pack_entry(int X, int Y, int a, int b, int w, int h) {
    if (X < -1 || X > w - 1 || Y < -1 || Y > h - 1) return REMAP_MISS;
    return (uint32_t)(X + 1) | ((uint32_t)(Y + 1) << 11) | ((uint32_t)a << 22) | ((uint32_t)b << 27);
}

// float coordinate -> fixed point as cv::convertMaps: saturate_cast<int>(v * 32) (round half to even; a value outside the int
// range, or NaN, becomes INT_MIN there, whose footprint misses every image)
__device__ __forceinline__ bool fixed_from_float(float v, int& q) {
    const float s = v * 32.0f;                                    // exact: a power of two
    if (!(s > -2147483648.0f && s < 2147483648.0f)) return false;
    q = __float2int_rn(s);
    return true;
}

__global__ void __launch_bounds__(256) remap_convert_kernel(int type, const uint8_t* __restrict__ m1, size_t s1,
                                                            const uint8_t* __restrict__ m2, size_t s2, int w, int h,
                                                            uint32_t* __restrict__ out, int pitch) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= pitch || y >= h) return;
    uint32_t e = REMAP_MISS;
    if (x < w) {
        if (type == OV2_MAP_16SC2) {
            const short2 xy = reinterpret_cast<const short2*>(m1 + (size_t)y * s1)[x];
            const unsigned f = reinterpret_cast<const uint16_t*>(m2 + (size_t)y * s2)[x];
            e = pack_entry(xy.x, xy.y, (int)(f & 31u), (int)((f >> 5) & 31u), w, h);
        } else {
            const float fx = reinterpret_cast<const float*>(m1 + (size_t)y * s1)[x];
            const float fy = reinterpret_cast<const float*>(m2 + (size_t)y * s2)[x];
            int qx, qy;
            if (fixed_from_float(fx, qx) && fixed_from_float(fy, qy)) {
                // X = saturate_cast<short>(qx >> 5): a clamped value is far outside any image as well
                e = pack_entry(qx >> 5, qy >> 5, qx & 31, qy & 31, w, h);
            }
        }
    }
    out[(size_t)y * pitch + x] = e;
}

struct RemapArgs {
    const uint32_t* map; int mpitch;
    const uint8_t* src; long long spitch, sfstride;
    uint8_t* dst; long long dpitch, dfstride;
    int w, h, count, per_group;
};

__device__ __forceinline__ uint32_t remap_pixel(uint32_t e, const uint8_t* __restrict__ img, long long pitch, int w, int h) {
    if (e == REMAP_MISS) return 0u;
    const int X = (int)(e & 0x7FFu) - 1, Y = (int)((e >> 11) & 0x7FFu) - 1;
    const int a = (int)((e >> 22) & 31u), b = (int)(e >> 27);
    int p00, p01, p10, p11;
    if (X >= 0 && Y >= 0 && X + 1 < w && Y + 1 < h) {
        const uint8_t* r0 = img + (long long)Y * pitch + X;
        p00 = __ldg(r0); p01 = __ldg(r0 + 1);
        p10 = __ldg(r0 + pitch); p11 = __ldg(r0 + pitch + 1);
    } else {                                                       // footprint straddles the border: outside reads 0
        const bool x0 = X >= 0, x1 = X + 1 < w, y0 = Y >= 0, y1 = Y + 1 < h;
        const uint8_t* r0 = img + (long long)Y * pitch + X;
        p00 = x0 && y0 ? __ldg(r0) : 0;
        p01 = x1 && y0 ? __ldg(r0 + 1) : 0;
        p10 = x0 && y1 ? __ldg(r0 + pitch) : 0;
        p11 = x1 && y1 ? __ldg(r0 + pitch + 1) : 0;
    }
    const int s = (32 - a) * ((32 - b) * p00 + b * p10) + a * ((32 - b) * p01 + b * p11);
    return (uint32_t)((s + 512) >> 10);
}

__global__ void __launch_bounds__(RT_X* RT_Y, 4) remap_kernel(RemapArgs A) {
    const int x = (blockIdx.x * RT_X + threadIdx.x) * 4;
    const int y = blockIdx.y * RT_Y + threadIdx.y;
    if (x >= A.w || y >= A.h) return;
    const uint4 m = __ldg(reinterpret_cast<const uint4*>(A.map + (size_t)y * A.mpitch + x));
    const int f0 = blockIdx.z * A.per_group;
    const int f1 = min(f0 + A.per_group, A.count);
    const bool full = x + 4 <= A.w;
    for (int f = f0; f < f1; ++f) {
        const uint8_t* img = A.src + A.sfstride * f;
        uint8_t* drow = A.dst + A.dfstride * f + A.dpitch * y + x;
        const uint32_t out = remap_pixel(m.x, img, A.spitch, A.w, A.h) | (remap_pixel(m.y, img, A.spitch, A.w, A.h) << 8) |
                             (remap_pixel(m.z, img, A.spitch, A.w, A.h) << 16) | (remap_pixel(m.w, img, A.spitch, A.w, A.h) << 24);
        if (full && (reinterpret_cast<uintptr_t>(drow) & 3) == 0) {
            *reinterpret_cast<uint32_t*>(drow) = out;
        } else {
            for (int k = 0; k < 4 && x + k < A.w; ++k) drow[k] = (uint8_t)(out >> (8 * k));
        }
    }
}

}  // namespace

// everything on the device already: `count` frames of src -> dst through `map`
ov2_status ov2_remap_device(ov2_ctx* ctx, const ov2_remap_map* map, const uint8_t* src, size_t spitch, size_t sfstride, uint8_t* dst,
                            size_t dpitch, size_t dfstride, int count) {
    RemapArgs A;
    A.map = map->entries; A.mpitch = map->pitch;
    A.src = src; A.spitch = (long long)spitch; A.sfstride = (long long)sfstride;
    A.dst = dst; A.dpitch = (long long)dpitch; A.dfstride = (long long)dfstride;
    A.w = map->w; A.h = map->h; A.count = count;
    const int tiles = div_up(map->w, R_TILE_W) * div_up(map->h, RT_Y);
    int groups = div_up(8 * ctx->sm_count, tiles);                // about 8 CTAs per SM in flight
    if (groups > count) groups = count;
    if (groups < 1) groups = 1;
    A.per_group = div_up(count, groups);
    groups = div_up(count, A.per_group);
    const dim3 grid(div_up(map->w, R_TILE_W), div_up(map->h, RT_Y), groups);
    OV2_LAUNCH(ctx, "remap_kernel", remap_kernel<<<grid, dim3(RT_X, RT_Y), 0, ctx->stream>>>(A));
    return OV2_OK;
}

extern "C" ov2_status ov2_remap_create(ov2_ctx* ctx, int map_type, int width, int height, const void* map1, size_t map1_stride,
                                       const void* map2, size_t map2_stride, ov2_remap_map** out) {
    if (!ctx || !out || !map1 || !map2 || width <= 0 || height <= 0 || (map_type != OV2_MAP_16SC2 && map_type != OV2_MAP_32FC1))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap_create: bad arguments");
    const size_t e1 = 4, e2 = map_type == OV2_MAP_16SC2 ? 2 : 4;     // bytes per map1 / map2 element
    if (map1_stride < (size_t)width * e1 || map2_stride < (size_t)width * e2 || (map1_stride % e1) != 0 || (map2_stride % e2) != 0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap_create: bad map strides");
    *out = nullptr;
    if (width > REMAP_MAX_SIDE || height > REMAP_MAX_SIDE)
        return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_remap_create: images larger than 2046 px per side are not supported");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    const void* d1 = nullptr;
    const void* d2 = nullptr;
    if ((st = ov2_stage_in(ctx, map1, map1_stride * (size_t)(height - 1) + (size_t)width * e1, &d1)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, map2, map2_stride * (size_t)(height - 1) + (size_t)width * e2, &d2)) != OV2_OK) return st;
    if (((reinterpret_cast<uintptr_t>(d1) % e1) | (reinterpret_cast<uintptr_t>(d2) % e2)) != 0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap_create: misaligned device maps");
    ov2_remap_map* m = new ov2_remap_map();
    m->device = ctx->device;
    m->w = width; m->h = height;
    m->pitch = (width + 3) & ~3;
    cudaError_t e = cudaMalloc(&m->entries, (size_t)m->pitch * height * sizeof(uint32_t));
    if (e != cudaSuccess) {
        delete m;
        return ov2_fail(ctx, OV2_ERR_NOMEM, "ov2_remap_create: cudaMalloc", e);
    }
    remap_convert_kernel<<<dim3(div_up(m->pitch, 256), height), 256, 0, ctx->stream>>>(map_type, (const uint8_t*)d1, map1_stride,
                                                                                     (const uint8_t*)d2, map2_stride, width, height,
                                                                                     m->entries, m->pitch);
    ctx->launches++;
    e = cudaGetLastError();
    if (e != cudaSuccess) {
        cudaFree(m->entries);
        delete m;
        return ov2_fail(ctx, OV2_ERR_CUDA, "remap_convert_kernel", e);
    }
    // the map is built once per camera: finish it here, so that the caller may free its maps on return
    if (!ctx->batch && (st = ov2_wait_stream(ctx)) != OV2_OK) {
        cudaFree(m->entries);
        delete m;
        return st;
    }
    *out = m;
    return OV2_OK;
}

extern "C" void ov2_remap_destroy(ov2_remap_map* map) {
    if (!map) return;
    cudaSetDevice(map->device);
    cudaDeviceSynchronize();             // launches of any context may still read it
    cudaFree(map->entries);
    delete map;
}

extern "C" ov2_status ov2_remap(ov2_ctx* ctx, const ov2_remap_map* map, const uint8_t* src, size_t src_row_stride,
                                size_t src_frame_stride, uint8_t* dst, size_t dst_row_stride, size_t dst_frame_stride, int count) {
    if (!ctx || !map || !src || !dst || count <= 0 || src_row_stride < (size_t)map->w || dst_row_stride < (size_t)map->w ||
        (count > 1 && (src_frame_stride < src_row_stride * (size_t)map->h || dst_frame_stride < dst_row_stride * (size_t)map->h)))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap: bad arguments");
    if (map->device != ctx->device) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap: map lives on another device");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    const size_t sb = src_frame_stride * (size_t)(count - 1) + src_row_stride * (size_t)(map->h - 1) + (size_t)map->w;
    const size_t db = dst_frame_stride * (size_t)(count - 1) + dst_row_stride * (size_t)(map->h - 1) + (size_t)map->w;
    const void* d = nullptr;
    void* o = nullptr;
    if ((st = ov2_stage_in(ctx, src, sb, &d)) != OV2_OK) return st;
    // a host destination is staged as one span and copied back whole: when its rows or frames have gaps, copy the span in
    // first so that the bytes between them (other pixels of a ROI's parent image) come back unchanged
    const bool dhost = !ov2_is_device_ptr(dst);
    const bool gaps = dst_row_stride != (size_t)map->w || (count > 1 && dst_frame_stride != dst_row_stride * (size_t)map->h);
    if ((st = ov2_stage_out(ctx, dst, db, &o, dhost && gaps)) != OV2_OK) return st;
    if (!dhost && d == (const void*)o) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_remap: device dst may not alias src");
    if ((st = ov2_remap_device(ctx, map, (const uint8_t*)d, src_row_stride, src_frame_stride, (uint8_t*)o, dst_row_stride,
                               dst_frame_stride, count)) != OV2_OK)
        return st;
    return ov2_end(ctx);
}

// ov2_pyr_build through a rectification map: the unrectified images (host: uploaded once into scratch; device: read in place)
// are remapped into the pyramid's OWN level 0, then its levels are built.
extern "C" ov2_status ov2_pyr_build_remap(ov2_ctx* ctx, ov2_pyr* p, const ov2_remap_map* map, const uint8_t* images, size_t row_stride,
                                          size_t frame_stride, int first, int count) {
    if (!ctx || !p || !map || !images || first < 0 || count <= 0 || first + count > p->batch || row_stride < (size_t)p->w[0] ||
        (count > 1 && frame_stride < row_stride * (size_t)p->h[0]))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build_remap: bad arguments");
    if (map->w != p->w[0] || map->h != p->h[0]) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build_remap: map and pyramid sizes differ");
    if (map->device != ctx->device) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build_remap: map lives on another device");
    if (p->l0_mode == 2) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build_remap: pyramid aliases device images");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    if (!p->own[0]) {
        OV2_CUDA(ctx, cudaMalloc(&p->own[0], p->fstride[0] * (size_t)p->batch));
        p->l0 = p->own[0]; p->l0_pitch = p->pitch[0]; p->l0_fstride = p->fstride[0]; p->l0_mode = 1;
    }
    const size_t sb = frame_stride * (size_t)(count - 1) + row_stride * (size_t)(p->h[0] - 1) + (size_t)p->w[0];
    const void* d = nullptr;
    if ((st = ov2_stage_in(ctx, images, sb, &d)) != OV2_OK) return st;
    if ((st = ov2_remap_device(ctx, map, (const uint8_t*)d, row_stride, frame_stride, p->own[0] + p->fstride[0] * (size_t)first,
                               p->pitch[0], p->fstride[0], count)) != OV2_OK)
        return st;
    if ((st = ov2_pyr_make_levels(ctx, p, first, count)) != OV2_OK) return st;
    return ov2_end(ctx);
}
