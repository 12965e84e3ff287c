// 8f-3: the stereo prior of rectified configurations - FeatureTracker::getLineMinSAD for a whole batch of keypoints.
//
// Reference behaviour replaced: FeatureTracker::getLineMinSAD (/root/reference/src/feature_tracker.cpp:138-204), which
// MapManager::stereoMatching calls once per 2-D keypoint of a keyframe (/root/reference/src/map_manager.cpp:417-431,
// `bdo_stereo_rect` configurations) on the coarsest pyramid level: take the sub-pixel 7 x 7 patch around the left
// keypoint (cv::getRectSubPix), slide a 7 x 7 target along the same row of the right image in unit steps starting at
// the keypoint's column (downwards when `bgoleft`), keep the column with the smallest mean absolute difference.
//
// One warp per keypoint; lane l evaluates the candidates l, l + 32, ... with exactly the reference's arithmetic:
//   * the window shrink near the borders (the reference's int += float compound assignments truncate),
//   * cv::getRectSubPix 8u -> 8u as OpenCV's template computes it (16-bit fixed-point bilinear weights
//     cvRound(w * 65536), (sum + 2^15) >> 16, replicated border) - the same restatement the host shim
//     (host/feature_tracker.cpp) and oracle/image_ref.py::get_rect_subpix_u8_ref use,
//   * candidate columns c_k formed by k repeated float subtractions / additions of 1 (the additions round when c
//     crosses a power of two, so they are replayed, not multiplied out),
//   * l1err = (float)sum / nbwinpx in float, strict `<` against the running minimum in scan order: the first of equal
//     minima wins (warp arg-min over (error, k)), a minimum of 255 or more leaves xprior = -1.
#include <climits>
#include "ov2_common.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int WARPS = 4;
constexpr int MAX_WS = 15;
// The reference's border rule can GROW the half window (halfwin += x + halfwin - cols - 1 is positive within one pixel of
// the right / bottom edge, feature_tracker.cpp:155-160).  The sum is taken in float: for x just below cols, x + h can round
// up to exactly cols + h, so each edge test takes h to 2 h - 1 (not 2 h - 2), and an in-image point reaches 4 h0 - 3 after
// both tests (h0 = nwinsize / 2; 25 for window 15, e.g. (93.99999, 59.999996) on a 94 x 60 level).  Points past the right
// or bottom edge can grow further; they get (-1, 255) once the half window exceeds this bound.
constexpr int MAX_HW = 4 * (MAX_WS / 2) - 3;             // 25
constexpr int MAX_PATCH = (2 * MAX_HW + 1) * (2 * MAX_HW + 1);

struct SadArgs {
    PyrView L, R;
    int level;
    int n;
    const int32_t* frame_idx; int first_frame, per_frame;
    const float2* pts;
    int nwinsize, goleft;
    float* xprior;
    float* l1err;
};

struct Sampler {
    int ipx, ipy, a11, a12, a21, a22;
};

__device__ __forceinline__ Sampler make_sampler(int ws, float cx, float cy) {
    Sampler s;
    cx -= (float)(ws - 1) * 0.5f;
    cy -= (float)(ws - 1) * 0.5f;
    s.ipx = __float2int_rd(cx);
    s.ipy = __float2int_rd(cy);
    const float a = cx - (float)s.ipx, b = cy - (float)s.ipy;
    s.a11 = __float2int_rn((1.f - a) * (1.f - b) * 65536.f);
    s.a12 = __float2int_rn(a * (1.f - b) * 65536.f);
    s.a21 = __float2int_rn((1.f - a) * b * 65536.f);
    s.a22 = __float2int_rn(a * b * 65536.f);
    return s;
}

__device__ __forceinline__ int sample(const uint8_t* img, int pitch, int w, int h, const Sampler& s, int i, int j) {
    const int x0 = clampi(s.ipx + j, 0, w - 1), x1 = clampi(s.ipx + j + 1, 0, w - 1);
    const int y0 = clampi(s.ipy + i, 0, h - 1), y1 = clampi(s.ipy + i + 1, 0, h - 1);
    const uint8_t* r0 = img + (size_t)y0 * pitch;
    const uint8_t* r1 = img + (size_t)y1 * pitch;
    const int v = (int)__ldg(r0 + x0) * s.a11 + (int)__ldg(r0 + x1) * s.a12 + (int)__ldg(r1 + x0) * s.a21 + (int)__ldg(r1 + x1) * s.a22;
    return (v + (1 << 15)) >> 16;
}

__global__ void __launch_bounds__(WARPS * 32) line_min_sad_kernel(SadArgs A) {
    __shared__ uint8_t spatch[WARPS][MAX_PATCH + 3];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * WARPS + warp;
    if (i >= A.n) return;
    const float2 pt = A.pts[i];
    const int lv = A.level;
    const int cols = A.R.w[lv], rows = A.R.h[lv];
    float xprior = -1.f, minsad = 255.f;
    const float x = pt.x, y = pt.y;
    int halfwin = A.nwinsize / 2;
    if (x - (float)halfwin < 0.f) halfwin = (int)((float)halfwin + (x - (float)halfwin));
    if (x + (float)halfwin >= (float)cols) halfwin = (int)((float)halfwin + (x + (float)halfwin - (float)cols - 1.f));
    if (y - (float)halfwin < 0.f) halfwin = (int)((float)halfwin + (y - (float)halfwin));
    if (y + (float)halfwin >= (float)rows) halfwin = (int)((float)halfwin + (y + (float)halfwin - (float)rows - 1.f));
    // x < 0 marks an empty slot (as in the other operators); NaN coordinates fall out of every comparison above
    if (halfwin <= 0 || halfwin > MAX_HW || !(x >= 0.f)) {
        if (lane == 0) { A.xprior[i] = -1.f; A.l1err[i] = 255.f; }
        return;
    }
    const int frame = A.frame_idx ? A.frame_idx[i] : A.first_frame + i / A.per_frame;
    const uint8_t* iml = A.L.lvl[lv] + A.L.fstride[lv] * frame;
    const uint8_t* imr = A.R.lvl[lv] + A.R.fstride[lv] * frame;
    const int lp = A.L.pitch[lv], rp = A.R.pitch[lv];
    const int lw = A.L.w[lv], lh = A.L.h[lv];
    const int ws = 2 * halfwin + 1, npx = ws * ws;
    uint8_t* patch = spatch[warp];
    {
        const Sampler sp = make_sampler(ws, x, y);
        for (int p = lane; p < npx; p += 32) {
            const int r = p / ws, c = p - r * ws;
            patch[p] = (uint8_t)sample(iml, lp, lw, lh, sp, r, c);
        }
    }
    __syncwarp();
    // candidate k of this lane: c = x -/+ 1 applied k times
    float c = x;
    for (int k = 0; k < lane; ++k) c = A.goleft ? c - 1.f : c + 1.f;
    int best_s = INT_MAX, best_k = INT_MAX;
    float best_c = -1.f;
    const float fhw = (float)halfwin, fend = (float)(cols - halfwin);
    for (int k = lane;; k += 32) {
        const bool in = A.goleft ? (c >= fhw) : (c < fend);
        if (!__any_sync(FULL, in)) break;        // the scan is monotone: once every lane is out, all later k are out
        if (in) {
            const Sampler sc = make_sampler(ws, c, y);
            int s = 0;
            for (int r = 0; r < ws; ++r)
                for (int q = 0; q < ws; ++q) s += abs((int)patch[r * ws + q] - sample(imr, rp, cols, rows, sc, r, q));
            if (s < best_s) { best_s = s; best_k = k; best_c = c; }   // strict: the lane's first minimum in scan order
        }
        for (int t = 0; t < 32; ++t) c = A.goleft ? c - 1.f : c + 1.f;
    }
    // warp arg-min over (sum, k): the mean error is strictly monotone in the integer sum (sums < 2^24, one divisor)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int os = __shfl_xor_sync(FULL, best_s, o), ok = __shfl_xor_sync(FULL, best_k, o);
        const float oc = __shfl_xor_sync(FULL, best_c, o);
        if (os < best_s || (os == best_s && ok < best_k)) { best_s = os; best_k = ok; best_c = oc; }
    }
    if (best_k != INT_MAX) {
        const float e = __fdiv_rn((float)best_s, (float)npx);
        if (e < minsad) { minsad = e; xprior = best_c; }
    }
    if (lane == 0) { A.xprior[i] = xprior; A.l1err[i] = minsad; }
}

}  // namespace

extern "C" ov2_status ov2_line_min_sad(ov2_ctx* ctx, const ov2_pyr* left, const ov2_pyr* right, int level, int n,
                                       const int32_t* frame_idx, int first_frame, int per_frame, const float* pts, int nwinsize,
                                       int goleft, float* xprior_out, float* l1err_out) {
    if (!ctx || !left || !right || n < 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: bad arguments");
    if (n == 0) return OV2_OK;
    if (!pts || !xprior_out || !l1err_out || (!frame_idx && per_frame <= 0)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: null array");
    if (nwinsize % 2 == 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: getLineMinSAD requires an odd window size");   // feature_tracker.cpp:144-147
    if (nwinsize < 1 || nwinsize > MAX_WS) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_line_min_sad: window sizes up to 15 are built");
    if (level < 0 || level >= left->nlev || level >= right->nlev || level > 3)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: pyramid level not built");
    if (!left->l0 || !right->l0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: pyramids not built");
    if (!frame_idx && (first_frame < 0 || first_frame + (n + per_frame - 1) / per_frame > left->batch ||
                       first_frame + (n + per_frame - 1) / per_frame > right->batch))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_line_min_sad: more frames than pyramid slots");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    SadArgs A;
    A.L = make_view(left);
    A.R = make_view(right);
    A.level = level;
    A.n = n;
    A.first_frame = first_frame;
    A.per_frame = per_frame;
    A.nwinsize = nwinsize;
    A.goleft = goleft ? 1 : 0;
    if ((st = ov2_stage_in(ctx, frame_idx, (size_t)n, A.frame_idx)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, pts, (size_t)n, A.pts)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, xprior_out, (size_t)n, A.xprior)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, l1err_out, (size_t)n, A.l1err)) != OV2_OK) return st;
    OV2_LAUNCH(ctx, "line_min_sad_kernel", line_min_sad_kernel<<<div_up(n, WARPS), WARPS * 32, 0, ctx->stream>>>(A));
    return ov2_end(ctx);
}
