// B: binary descriptors, one warp per keypoint.
//
// Reference behaviour replaced: FeatureExtractor::describeBRIEF, non-contrib branch
// cv::ORB::create(500, 1., 0).compute(im, kps, descs) (/root/reference/src/feature_extractor.cpp:
// 224-285, :245).  For the keypoints the reference passes (size 1, angle -1, octave 0) that is:
//   drop keypoints whose rounded centre is closer than 31 px to the border,
//   smooth the image with a float32 separable 7-tap Gaussian (sigma 2) and round to u8,
//   256 intensity comparisons on the ORB pattern around c = cvRound(pt)   (SURVEY.md A.5).
// For sparse keypoint sets, instead of smoothing the whole image (2 x W x H bytes of traffic per
// frame) each warp smooths only the 26x26 window the pattern touches, from a 32x32 raw window, in
// shared memory, with exactly OpenCV's float operation order (rows: sequential FMA chain; columns:
// symmetric pairs + FMA; pinned bit-exact by oracle/image_ref.py::smooth7_ref against cv2).
// Keypoints are >= 31 px from the border, so the 32x32 window never needs the REFLECT_101 border.
// Dense fixed-stride sets, whose windows would smooth every reachable pixel several times over (C2's
// 1024 keypoints per 640x480 frame: 2.6 times), take the dense path instead: one smoothing pass per
// frame into a scratch plane, then a gather per keypoint (ov2_describe picks by density).
//
// The descriptor is DATA-driven (ov2_describe_config): mode OV2_DESC_ORB_FALLBACK is the above; mode
// OV2_DESC_BRIEF32 is the reference's DEFAULT build (CMakeLists.txt:12 WITH_OPENCV_CONTRIB,
// feature_extractor.cpp:242-243 cv::xfeatures2d::BriefDescriptorExtractor::create()): 256 comparisons of 9 x 9
// box sums (an integral-image lookup in opencv_contrib's brief.cpp, `smoothedSum`) at the test pairs of
// generated_32.i around (int)(pt + 0.5), first test in bit 7 of its byte, keypoints whose rounded centre is
// closer than PATCH_SIZE/2 + KERNEL_SIZE/2 = 28 px to the border dropped.  The 256 pairs ship only with
// opencv_contrib (not in this image): the caller loads them (scripts/brief_table_from_contrib.py turns
// generated_32.i into the table), the kernel (`describe_box_kernel`) is table-agnostic.
#include "ov2_common.cuh"
#include "../../include/ov2_orb_pattern.h"

namespace {

constexpr int WARPS = 4;

__device__ __align__(16) signed char g_pat[256][4];   // global (not __constant__): every lane reads its own 8 pairs
__constant__ float c_gk[7];

struct DescArgs {
    const uint8_t* img; int w, h, pitch; long long fstride;
    int n;
    const int32_t* frame_idx; int first_frame, per_frame;
    const float2* pts;
    uint8_t* desc; uint8_t* valid;
};

// The two passes of the 7-tap smoothing, shared by the per-window and the dense kernels so that both
// produce the same bytes.  Row: output at the centre tap x3, sequential FMA chain exactly as OpenCV's
// float row filter evaluates it.
__device__ __forceinline__ float smooth_row7(float x0, float x1, float x2, float x3, float x4, float x5, float x6,
                                             float k0, float k1, float k2, float k3) {
    float acc = x0 * k0;
    acc = __fmaf_rn(x1, k1, acc);
    acc = __fmaf_rn(x2, k2, acc);
    acc = __fmaf_rn(x3, k3, acc);
    acc = __fmaf_rn(x4, k2, acc);
    acc = __fmaf_rn(x5, k1, acc);
    acc = __fmaf_rn(x6, k0, acc);
    return acc;
}

// Column: output at the centre tap y3, symmetric pairs + FMA as OpenCV's float column filter, then
// saturate_cast<uchar> (round half to even, clamp).  The clamp comes first, which gives the same integer
// because rint is monotone and 0, 255 are integers; adding 1.5 * 2^23 then rounds to an integer in the low
// mantissa bits (exact below 2^22), so the conversion stays on the FP32 pipe.  Returns the value in bits 0..7.
__device__ __forceinline__ unsigned smooth_col7(float y0, float y1, float y2, float y3, float y4, float y5, float y6,
                                                float k0, float k1, float k2, float k3) {
    float acc = y3 * k3;
    acc = __fmaf_rn(y2 + y4, k2, acc);
    acc = __fmaf_rn(y1 + y5, k1, acc);
    acc = __fmaf_rn(y0 + y6, k0, acc);
    acc = fminf(fmaxf(acc, 0.f), 255.f);
    return __float_as_uint(acc + 12582912.f) & 255u;
}

// ORB-fallback border rule, KeyPointsFilter::runByImageBorder(kps, size, 31) on the rounded point; x < 0
// marks an empty slot.  Writes the zero descriptor and valid = 0 for a dropped point.
__device__ __forceinline__ bool orb_drop(const DescArgs& A, int i, float2 pt, int cx, int cy, int lane) {
    if (pt.x < 0.f || cx < 31 || cy < 31 || cx >= A.w - 31 || cy >= A.h - 31) {
        A.desc[(size_t)i * 32 + lane] = 0;
        if (lane == 0) A.valid[i] = 0;
        return true;
    }
    return false;
}

// 8 tests per lane -> descriptor byte `lane`; at(dx, dy) reads the smoothed pixel at offset (dx, dy) from the
// rounded centre
template <class At>
__device__ __forceinline__ unsigned orb_byte(int lane, At at) {
    const int4 pa = __ldg(reinterpret_cast<const int4*>(&g_pat[lane * 8][0]));
    const int4 pb = __ldg(reinterpret_cast<const int4*>(&g_pat[lane * 8 + 4][0]));
    const int pw[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
    unsigned byte = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int t0 = (int)(signed char)(pw[k] & 255), t1 = (int)(signed char)((pw[k] >> 8) & 255);
        const int t2 = (int)(signed char)((pw[k] >> 16) & 255), t3 = (int)(signed char)((pw[k] >> 24) & 255);
        byte |= (unsigned)(at(t0, t1) < at(t2, t3)) << k;
    }
    return byte;
}

__global__ void __launch_bounds__(WARPS * 32) describe_kernel(DescArgs A) {
    __shared__ float sraw[WARPS][32 * 33];   // 32x32 raw window as float (+1 pad: conflict-free rows); row-filtered IN PLACE
    __shared__ uint8_t ssm[WARPS][26 * 28];  // 26 x 26 smoothed (+2 pad)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + warp;
    if (i >= A.n) return;
    const float2 pt = A.pts[i];
    const int cx = __float2int_rn(pt.x), cy = __float2int_rn(pt.y);
    uint8_t* dout = A.desc + (size_t)i * 32;
    if (orb_drop(A, i, pt, cx, cy, lane)) return;
    const int frame = A.frame_idx ? A.frame_idx[i] : A.first_frame + i / A.per_frame;
    const uint8_t* img = A.img + A.fstride * frame + (size_t)(cy - 16) * A.pitch + (cx - 16);
    float* raw = sraw[warp];
    float* row = raw;   // the row filter overwrites column c only after its taps c..c+6 sit in registers
    uint8_t* sm = ssm[warp];
    // raw window rows cy-16..cy+15, cols cx-16..cx+15 (lane = column): 32 coalesced 32-byte reads
#pragma unroll 8
    for (int r = 0; r < 32; ++r) raw[r * 33 + lane] = (float)__ldg(img + (size_t)r * A.pitch + lane);
    __syncwarp();
    const float k0 = c_gk[0], k1 = c_gk[1], k2 = c_gk[2], k3 = c_gk[3];
    // row filter, lane = row: output col c (0..25) <-> image col cx-13+c, taps raw cols c..c+6
    {
        const float* p = raw + lane * 33;
        float x0 = p[0], x1 = p[1], x2 = p[2], x3 = p[3], x4 = p[4], x5 = p[5];
#pragma unroll
        for (int c = 0; c < 26; ++c) {
            const float x6 = p[c + 6];
            row[lane * 33 + c] = smooth_row7(x0, x1, x2, x3, x4, x5, x6, k0, k1, k2, k3);
            x0 = x1; x1 = x2; x2 = x3; x3 = x4; x4 = x5; x5 = x6;
        }
    }
    __syncwarp();
    // column filter, lane = column: output row q (0..25) <-> image row cy-13+q, taps rows q..q+6
    if (lane < 26) {
        const float* p = row + lane;
        float y0 = p[0], y1 = p[33], y2 = p[2 * 33], y3 = p[3 * 33], y4 = p[4 * 33], y5 = p[5 * 33];
#pragma unroll
        for (int q = 0; q < 26; ++q) {
            const float y6 = p[(q + 6) * 33];
            sm[q * 28 + lane] = (uint8_t)smooth_col7(y0, y1, y2, y3, y4, y5, y6, k0, k1, k2, k3);
            y0 = y1; y1 = y2; y2 = y3; y3 = y4; y4 = y5; y5 = y6;
        }
    }
    __syncwarp();
    dout[lane] = (uint8_t)orb_byte(lane, [&](int dx, int dy) { return (int)sm[(dy + 13) * 28 + (dx + 13)]; });
    if (lane == 0) A.valid[i] = 1;
}


// ---- Dense path for keypoint sets that cover each frame several times over (see ov2_describe): the smoothed
// image is computed once per frame into a plane, then every keypoint reads its 512 test pixels from it.
// Plane: same geometry as level 0 (pitch rounded up to 16 bytes), written only where a valid keypoint's pattern
// can reach (centres >= 31 px from the border, pattern radius 13): rows [18, h - 18) and a column band [16, ...)
// that covers [18, w - 18) in runs of SMOOTH_COLS.  The filter reaches 3 px, so every tap lies inside the image
// and no border handling is needed.  Needs w, h >= 63 (the smallest frame with a valid centre).
constexpr int SMOOTH_COLS = 8;    // output columns per thread (one 8-byte store per row)
constexpr int SMOOTH_ROWS = 16;   // output rows per thread (SMOOTH_ROWS + 6 row-filtered rows in registers)
constexpr int SMOOTH_THREADS = 128;

struct SmoothArgs {
    const uint8_t* img; int pitch; long long fstride;
    int first_frame, h;
    int ncs, nrs;                 // column runs and row runs per frame
    uint8_t* plane; int ppitch; long long pfstride;
};

__global__ void __launch_bounds__(SMOOTH_THREADS) desc_smooth_kernel(SmoothArgs S) {
    const int t = blockIdx.x * SMOOTH_THREADS + threadIdx.x;
    if (t >= S.ncs * S.nrs) return;
    const int cs = t % S.ncs, rs = t / S.ncs;
    const int x0 = 16 + SMOOTH_COLS * cs;
    // the last row run is pulled up to end at h - 18 (overlapping runs write the same bytes); rows read stay in
    // [15, h - 16)
    const int y0 = min(18 + SMOOTH_ROWS * rs, S.h - 18 - SMOOTH_ROWS);
    // taps of output columns x0 .. x0+7 are image columns x0-3 .. x0+10; read the 16 bytes x0-4 .. x0+11 as five
    // aligned words (the row and the pitch need not be aligned) and funnel-shift them into place.  x0+7 <= w - 12,
    // so every word lies inside the row.
    const uint8_t* src = S.img + S.fstride * (S.first_frame + (int)blockIdx.y) + (size_t)(y0 - 3) * S.pitch + (x0 - 4);
    uint8_t* dst = S.plane + S.pfstride * (int)blockIdx.y + (size_t)y0 * S.ppitch + x0;
    const float k0 = c_gk[0], k1 = c_gk[1], k2 = c_gk[2], k3 = c_gk[3];
    auto row_words = [&](int r, unsigned* wd) {
        const unsigned* wp = reinterpret_cast<const unsigned*>(((uintptr_t)src + (size_t)r * S.pitch) & ~(uintptr_t)3);
#pragma unroll
        for (int k = 0; k < 5; ++k) wd[k] = __ldg(wp + k);
    };
    unsigned nxt[5];              // words of the next row, loaded one row ahead of their use
    row_words(0, nxt);
    float win[7][SMOOTH_COLS];    // row-filtered rows y-3 .. y+3 of the next output row y
#pragma unroll
    for (int r = 0; r < SMOOTH_ROWS + 6; ++r) {
        const unsigned w0 = nxt[0], w1 = nxt[1], w2 = nxt[2], w3 = nxt[3], w4 = nxt[4];
        const unsigned s = (unsigned)(((uintptr_t)src + (size_t)r * S.pitch) & 3) * 8;
        if (r + 1 < SMOOTH_ROWS + 6) row_words(r + 1, nxt);
        const unsigned b[4] = {__funnelshift_r(w0, w1, s), __funnelshift_r(w1, w2, s), __funnelshift_r(w2, w3, s),
                               __funnelshift_r(w3, w4, s)};
        // byte j of b <-> image column x0-4+j; u8 -> float as (2^23 + v) - 2^23 (exact), on the FP32 pipe
        float f[16];
#pragma unroll
        for (int j = 1; j < 15; ++j)
            f[j] = __uint_as_float(__byte_perm(b[j >> 2], 0x4B000000u, 0x7650 | (j & 3))) - 8388608.f;
#pragma unroll
        for (int q = 0; q < 6; ++q)
#pragma unroll
            for (int c = 0; c < SMOOTH_COLS; ++c) win[q][c] = win[q + 1][c];
#pragma unroll
        for (int c = 0; c < SMOOTH_COLS; ++c)
            win[6][c] = smooth_row7(f[c + 1], f[c + 2], f[c + 3], f[c + 4], f[c + 5], f[c + 6], f[c + 7], k0, k1, k2, k3);
        if (r >= 6) {
            unsigned v[SMOOTH_COLS];
#pragma unroll
            for (int c = 0; c < SMOOTH_COLS; ++c)
                v[c] = smooth_col7(win[0][c], win[1][c], win[2][c], win[3][c], win[4][c], win[5][c], win[6][c], k0, k1, k2, k3);
            const uint2 o = make_uint2(v[0] | v[1] << 8 | v[2] << 16 | v[3] << 24, v[4] | v[5] << 8 | v[6] << 16 | v[7] << 24);
            *reinterpret_cast<uint2*>(dst + (size_t)(r - 6) * S.ppitch) = o;
        }
    }
}

struct DenseArgs {
    DescArgs d;
    const uint8_t* plane; int ppitch; long long pfstride;
};

// One warp per keypoint, lane = descriptor byte.  The 27 x 27 patch the pattern touches is first copied from the
// plane into shared memory as aligned words (4 rows x 8 words per load), so the 512 scattered byte reads hit
// shared memory instead of costing one L1 wavefront per distinct line.
__global__ void __launch_bounds__(WARPS * 32) describe_dense_kernel(DenseArgs D) {
    __shared__ unsigned spatch[WARPS][27 * 8];   // rows cy-13 .. cy+13, columns xb .. xb+31 (xb = (cx-13) & ~3)
    const DescArgs& A = D.d;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + warp;
    if (i >= A.n) return;
    const float2 pt = A.pts[i];
    const int cx = __float2int_rn(pt.x), cy = __float2int_rn(pt.y);
    if (orb_drop(A, i, pt, cx, cy, lane)) return;
    // plane rows are 16-byte aligned, so column alignment is address alignment; xb + 31 <= cx + 18 < pitch
    const int xb = (cx - 13) & ~3;
    const uint8_t* base = D.plane + D.pfstride * (i / A.per_frame) + (size_t)(cy - 13) * D.ppitch + xb;
    unsigned* patch = spatch[warp];
#pragma unroll
    for (int r = lane >> 3; r < 27; r += 4)
        patch[r * 8 + (lane & 7)] = __ldg(reinterpret_cast<const unsigned*>(base + (size_t)r * D.ppitch) + (lane & 7));
    __syncwarp();
    const uint8_t* pb = reinterpret_cast<const uint8_t*>(patch) + 13 * 32 + (cx - xb);
    A.desc[(size_t)i * 32 + lane] = (uint8_t)orb_byte(lane, [&](int dx, int dy) { return (int)pb[dy * 32 + dx]; });
    if (lane == 0) A.valid[i] = 1;
}


// ---- BRIEF-32 (box-smoothed tests): one warp per keypoint.
// raw  : 57 x 57 window (rows cy-28 .. cy+28), pitch 60 bytes
// hs   : horizontal 9-sums, hs[r][c] = sum raw[r][c .. c+8], c = 0..48 (centre column c+4), pitch 50 u16
// A test point (y, x), |y|, |x| <= 24, is the 9 x 9 box centred on raw (y+28, x+28):
//   S(y, x) = sum_{r = y+24 .. y+32} hs[r][x+24]      (exact integers, <= 81 * 255)
constexpr int BW = 57, BRAW_PITCH = 60, BHS_W = 49, BHS_PITCH = 50;

struct BoxArgs {
    DescArgs d;
    const signed char* table;   // [256][4] = (y0, x0, y1, x1) of SMOOTHED(y0, x0) < SMOOTHED(y1, x1), generated_32.i order
};

__global__ void __launch_bounds__(WARPS * 32) describe_box_kernel(BoxArgs B) {
    __shared__ __align__(4) uint8_t sraw[WARPS][BW * BRAW_PITCH];
    __shared__ __align__(4) unsigned short shs[WARPS][BW * BHS_PITCH];
    const DescArgs& A = B.d;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + warp;
    if (i >= A.n) return;
    const float2 pt = A.pts[i];
    uint8_t* dout = A.desc + (size_t)i * 32;
    // KeyPointsFilter::runByImageBorder(kps, size, 28) tests the cvRound'ed point
    const int rx = __float2int_rn(pt.x), ry = __float2int_rn(pt.y);
    if (pt.x < 0.f || rx < 28 || ry < 28 || rx >= A.w - 28 || ry >= A.h - 28) {
        dout[lane] = 0;
        if (lane == 0) A.valid[i] = 0;
        return;
    }
    // smoothedSum: img_x = (int)(pt.x + 0.5) + x  (truncation of a double sum; pt >= 27.5 here so floor == trunc)
    const int cx = (int)((double)pt.x + 0.5), cy = (int)((double)pt.y + 0.5);
    const int frame = A.frame_idx ? A.frame_idx[i] : A.first_frame + i / A.per_frame;
    const uint8_t* img = A.img + A.fstride * frame;
    uint8_t* raw = sraw[warp];
    unsigned short* hs = shs[warp];
    // cx can exceed the rounded centre by one at a .5 tie (window one column / row past the image when W - 29 is
    // even): those taps are clamped to the last column / row (OpenCV reads the integral image out of its row there)
    for (int r = 0; r < BW; ++r) {
        int y = cy - 28 + r;
        y = y > A.h - 1 ? A.h - 1 : y;
        const uint8_t* rowp = img + (size_t)y * A.pitch;
        int x0 = cx - 28 + lane, x1 = x0 + 32;
        x0 = x0 > A.w - 1 ? A.w - 1 : x0;
        x1 = x1 > A.w - 1 ? A.w - 1 : x1;
        raw[r * BRAW_PITCH + lane] = __ldg(rowp + x0);
        if (lane + 32 < BW) raw[r * BRAW_PITCH + lane + 32] = __ldg(rowp + x1);
    }
    __syncwarp();
    // horizontal sliding 9-sums, lane = row
    for (int r = lane; r < BW; r += 32) {
        const uint8_t* p = raw + r * BRAW_PITCH;
        unsigned short* o = hs + r * BHS_PITCH;
        int s = 0;
#pragma unroll
        for (int c = 0; c < 9; ++c) s += p[c];
        o[0] = (unsigned short)s;
#pragma unroll 8
        for (int c = 1; c < BHS_W; ++c) {
            s += (int)p[c + 8] - (int)p[c - 1];
            o[c] = (unsigned short)s;
        }
    }
    __syncwarp();
    // 8 tests per lane -> descriptor byte `lane`, first test in bit 7 (generated_32.i: (t0 << 7) + (t1 << 6) + ...)
    const int4 pa = __ldg(reinterpret_cast<const int4*>(B.table + (size_t)lane * 32));
    const int4 pb = __ldg(reinterpret_cast<const int4*>(B.table + (size_t)lane * 32 + 16));
    const int pw[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
    unsigned byte = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int y0 = (int)(signed char)(pw[k] & 255), x0 = (int)(signed char)((pw[k] >> 8) & 255);
        const int y1 = (int)(signed char)((pw[k] >> 16) & 255), x1 = (int)(signed char)((pw[k] >> 24) & 255);
        const unsigned short* pa0 = hs + (y0 + 24) * BHS_PITCH + (x0 + 24);
        const unsigned short* pb0 = hs + (y1 + 24) * BHS_PITCH + (x1 + 24);
        int a = 0, b = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r) {
            a += pa0[r * BHS_PITCH];
            b += pb0[r * BHS_PITCH];
        }
        byte |= (unsigned)(a < b) << (7 - k);
    }
    dout[lane] = (uint8_t)byte;
    if (lane == 0) A.valid[i] = 1;
}

bool g_tables_loaded[64] = {false};

// Dense path (smooth each frame once, then gather) when the keypoints' 26 x 26 windows cover the band a valid
// keypoint can reach, (w - 36) x (h - 36), at least DENSE_COVER times over.  The per-window kernel costs about
// per_frame * 26^2 smoothed pixels per frame, the dense one (w - 36)(h - 36) pixels plus a plane write and read.
// Measured with scripts/bench_describe.py (640 x 480, batch 256, H100 SXM 80GB at its 700 W limit, 1980 MHz):
// per-window / dense ms per call 0.145 / 0.151 at cover 1.29 (512 per frame), 0.212 / 0.175 at cover 1.94 (768),
// 0.279 / 0.199 at cover 2.58 (1024); the lines cross near cover 1.4.
constexpr float DENSE_COVER = 1.4f;

// Fixed-stride ORB-fallback calls only (ragged frame_idx calls keep the per-window kernel).
bool use_dense(const int32_t* frame_idx, int per_frame, int w, int h) {
    if (frame_idx || w < 63 || h < 63) return false;   // below 63 px no keypoint is valid
    return (double)per_frame * 26.0 * 26.0 >= (double)DENSE_COVER * (w - 36) * (h - 36);
}

}  // namespace


extern "C" ov2_status ov2_describe_config(ov2_ctx* ctx, int mode, const int8_t* pairs) {
    if (!ctx) return OV2_ERR_INVALID;
    if (mode == OV2_DESC_ORB_FALLBACK) {
        if (pairs) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe_config: the ORB-fallback pattern is built in (pass NULL)");
        ctx->desc_mode = OV2_DESC_ORB_FALLBACK;
        return OV2_OK;
    }
    if (mode != OV2_DESC_BRIEF32) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe_config: unknown descriptor mode");
    if (!pairs)
        return ov2_fail(ctx, OV2_ERR_INVALID,
                        "ov2_describe_config: BRIEF-32 needs the 256 test pairs of opencv_contrib's generated_32.i (not redistributed here)");
    int8_t host[1024];
    if (ov2_is_device_ptr(pairs)) OV2_CUDA(ctx, cudaMemcpy(host, pairs, 1024, cudaMemcpyDeviceToHost));
    else memcpy(host, pairs, 1024);
    for (int k = 0; k < 1024; ++k)
        if (host[k] < -24 || host[k] > 24)
            return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe_config: test offsets must lie in the 48 x 48 patch (|offset| <= 24)");
    if (!ctx->desc_table) OV2_CUDA(ctx, cudaMalloc(&ctx->desc_table, 1024));
    OV2_CUDA(ctx, cudaMemcpyAsync(ctx->desc_table, host, 1024, cudaMemcpyHostToDevice, ctx->stream));
    OV2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // `host` is a stack buffer
    ctx->desc_mode = OV2_DESC_BRIEF32;
    return OV2_OK;
}

extern "C" ov2_status ov2_describe(ov2_ctx* ctx, const ov2_pyr* pyr, int n, const int32_t* frame_idx, int first_frame, int per_frame,
                                   const float* pts, uint8_t* desc32_out, uint8_t* valid_out) {
    if (!ctx || !pyr || !pyr->l0 || n < 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe: bad arguments");
    if (n == 0) return OV2_OK;  // feature_extractor.cpp:226-229
    if (!pts || !desc32_out || !valid_out || (!frame_idx && per_frame <= 0))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe: null array");
    if (!frame_idx && (first_frame < 0 || first_frame + (n + per_frame - 1) / per_frame > pyr->batch))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_describe: more frames than pyramid slots");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    if (ctx->device < 64 && !g_tables_loaded[ctx->device]) {
        // cv::getGaussianKernel(7, 2, CV_32F) as exact float32 values (pinned in
        // tests/test_oracle_image.py against cv2.getGaussianKernel)
        const float kf[7] = {0x1.1f5f62p-4f, 0x1.0c70fcp-3f, 0x1.869472p-3f, 0x1.ba95c0p-3f,
                             0x1.869472p-3f, 0x1.0c70fcp-3f, 0x1.1f5f62p-4f};
        OV2_CUDA(ctx, cudaMemcpyToSymbol(c_gk, kf, sizeof(kf)));
        OV2_CUDA(ctx, cudaMemcpyToSymbol(g_pat, OV2_ORB_PATTERN, sizeof(OV2_ORB_PATTERN)));
        g_tables_loaded[ctx->device] = true;
    }
    DescArgs A;
    A.img = pyr->l0; A.w = pyr->w[0]; A.h = pyr->h[0]; A.pitch = (int)pyr->l0_pitch; A.fstride = (long long)pyr->l0_fstride;
    A.n = n; A.first_frame = first_frame; A.per_frame = per_frame;
    if ((st = ov2_stage_in(ctx, frame_idx, (size_t)n, A.frame_idx)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, pts, (size_t)n, A.pts)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, desc32_out, (size_t)32 * n, A.desc)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, valid_out, (size_t)n, A.valid)) != OV2_OK) return st;
    if (ctx->desc_mode == OV2_DESC_BRIEF32) {
        BoxArgs B;
        B.d = A;
        B.table = (const signed char*)ctx->desc_table;
        OV2_LAUNCH(ctx, "describe_box_kernel", describe_box_kernel<<<div_up(n, WARPS), WARPS * 32, 0, ctx->stream>>>(B));
    } else if (use_dense(frame_idx, per_frame, A.w, A.h)) {
        const int nframes = div_up(n, per_frame);
        DenseArgs D;
        D.d = A;
        D.ppitch = (A.w + 15) & ~15;
        D.pfstride = (long long)D.ppitch * A.h;
        uint8_t* pl = nullptr;
        if ((st = ov2_scratch(ctx, (size_t)D.pfstride * nframes, pl)) != OV2_OK) return st;
        D.plane = pl;
        SmoothArgs S;
        S.img = A.img; S.pitch = A.pitch; S.fstride = A.fstride;
        S.first_frame = first_frame; S.h = A.h;
        S.ncs = div_up(A.w - 34, SMOOTH_COLS);
        S.nrs = div_up(A.h - 36, SMOOTH_ROWS);
        S.plane = pl; S.ppitch = D.ppitch; S.pfstride = D.pfstride;
        OV2_LAUNCH(ctx, "desc_smooth_kernel",
                   desc_smooth_kernel<<<dim3(div_up(S.ncs * S.nrs, SMOOTH_THREADS), nframes), SMOOTH_THREADS, 0, ctx->stream>>>(S));
        OV2_LAUNCH(ctx, "describe_dense_kernel", describe_dense_kernel<<<div_up(n, WARPS), WARPS * 32, 0, ctx->stream>>>(D));
    } else {
        OV2_LAUNCH(ctx, "describe_kernel", describe_kernel<<<div_up(n, WARPS), WARPS * 32, 0, ctx->stream>>>(A));
    }
    return ov2_end(ctx);
}
