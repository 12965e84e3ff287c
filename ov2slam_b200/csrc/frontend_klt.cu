// K: forward/backward pyramidal Lucas-Kanade, one warp per keypoint, everything fused.
//
// Reference behaviour replaced: FeatureTracker::fbKltTracking
// (/root/reference/src/feature_tracker.cpp:35-137): forward cv::calcOpticalFlowPyrLK
// (USE_INITIAL_FLOW | LK_GET_MIN_EIGENVALS, maxLevel = nbpyrlvl) -> status / err / inBorder
// filter -> backward LK at level 0 -> forward-backward distance test.
//
// OpenCV's LK semantics (SURVEY.md A.3, pinned by oracle/image_ref.py::_lk_ref against cv2):
// 14-bit fixed-point bilinear weights, template / derivative patches as int16 (5 fractional bits
// on intensities), normal equations from *integer* window sums scaled by 2^-20 in float32.
// The window sums are reduced as integers across the warp (redux.sync, exact and order
// independent) and converted to float32 once; all float32 steps keep OpenCV's operation order
// (this file is compiled with -fmad=false so nothing is contracted into FMAs).
//
// Scharr derivatives are computed on the fly from a 12x12 8-bit neighbourhood (reflect-101 at
// the image edge, constant 0 outside the image - exactly the planes buildOpticalFlowPyramid
// would have materialised), so the tracker reads only the 8-bit pyramid.
//
// One kernel, fb_klt_kernel, instantiated for two window layouts: Win9 for the 9 x 9 window of every shipped configuration
// (three window pixels per lane, search taps packed in registers) and WinAny for every other window from 3 x 3 to 31 x 31
// (lane c owns window column c; template and staged image bytes in shared memory), profiled as fb_klt_win_kernel.
// ov2_fb_klt picks one from nwinsize.  Both run the same per-keypoint forward / backward logic, level and iteration
// control flow and float32 steps.
#include <climits>
#include "ov2_common.cuh"
#include "klt_setup.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;

struct KltArgs {
    PyrView prev, cur;
    int n;
    const int32_t* frame_idx;
    int first_frame, per_frame;
    const uint8_t* lvls;
    int lvl_all;
    const float2* kps;
    float2* priors;
    uint8_t* status;
    int max_iter;
    float eig_q;           // q < eig_q  <=>  minEig < LK_MIN_EIG, q the numerator of minEig (lk_eig_num)
    float ferr_q;          // q > ferr_q  <=>  minEig > ferr
    double fb_s;           // dx^2 + dy^2 > fb_s  <=>  sqrt(dx^2 + dy^2) > fb_dist (klt_setup.cuh, klt_fb_s)
    double eps2;           // epsilon^2 as OpenCV forms it (double)
    float eps_lo, eps_hi;  // float brackets of eps2: outside them the float evaluation of |delta|^2 decides
    int* work_counter;   // persistent launch: warps pull keypoint indices from this counter (null: one warp per index)
};

// exact 64-bit warp sum of per-lane int32 partials via two 32-bit redux ops
__device__ __forceinline__ long long warp_sum64(int s) {
    int lo = s & 0xFFFF;
    int hi = s >> 16;
    int slo = __reduce_add_sync(FULL, lo);
    int shi = __reduce_add_sync(FULL, hi);
    return ((long long)shi << 16) + (long long)slo;
}

// ---- OpenCV's float32 steps of one LK level, shared by both window layouts.  The weights, convergence and oscillation tests
// are macros rather than inline functions: as calls they change how fb_klt_kernel is scheduled.

// 14-bit bilinear weights of the sub-pixel offsets (a, b)
#define LK_WEIGHTS(a, b, iw00, iw01, iw10, iw11)                  \
    iw00 = __float2int_rn((1.f - (a)) * (1.f - (b)) * 16384.f);  \
    iw01 = __float2int_rn((a) * (1.f - (b)) * 16384.f);          \
    iw10 = __float2int_rn((1.f - (a)) * (b) * 16384.f);          \
    iw11 = 16384 - iw00 - iw01 - iw10

// The minimal eigenvalue of the normal matrix over a win x win window (the error LK_GET_MIN_EIGENVALS reports) is
// minEig = RN(q / (2 win^2)) with q this numerator.  A level whose minEig < LK_MIN_EIG or determinant < LK_MIN_DET
// (FLT_EPSILON) is dropped.  minEig is only ever compared, and RN(q / d) is monotone in q, so the trackers keep q and compare
// it against thresholds klt_launch computes for the call's win (KltArgs::eig_q, ferr_q): same decisions, no division.
// (double)minEig < 1e-4 <=> minEig < 0x1.a36e3p-14f, the smallest float >= 1e-4 (1e-4 is not a float)
__device__ __forceinline__ float lk_eig_num(float A11, float A12, float A22) {
    return A22 + A11 - __fsqrt_rn((A11 - A22) * (A11 - A22) + 4.f * A12 * A12);
}
constexpr float LK_MIN_EIG = 0x1.a36e3p-14f;
constexpr float LK_MIN_DET = 1.1920928955078125e-07f;

// the step from the mismatch sums, D = 1 / det
__device__ __forceinline__ float2 lk_step(float A11, float A12, float A22, float D, float b1, float b2) {
    return make_float2((A12 * b2 - A22 * b1) * D, (A12 * b1 - A11 * b2) * D);
}

// Declares bool conv: delta.ddot(delta) <= epsilon^2, a double comparison in OpenCV.  A float evaluation (relative error
// < 2e-7) decides it except within 1e-6 of the threshold (eps_lo .. eps_hi), where the double expression is evaluated.
#define LK_CONVERGED(conv, delta, eps2, eps_lo, eps_hi)                                                        \
    const float conv##_q = (delta).x * (delta).x + (delta).y * (delta).y;                                        \
    bool conv = conv##_q < (eps_lo);                                                                             \
    if (!conv && !(conv##_q > (eps_hi)))                                                                         \
    conv = (double)(delta).x * (double)(delta).x + (double)(delta).y * (double)(delta).y <= (eps2)

// (double)|f| < 0.01  <=>  |f| <= 0.01f: 0.01f = 0.00999999977... is the largest float below 0.01
#define LK_OSCILLATES(delta, prev) (fabsf((delta).x + (prev).x) <= 0.01f && fabsf((delta).y + (prev).y) <= 0.01f)

// The lane's search taps for the window origin (jx, jy): rows jy + lane_row and +1, columns jx + lane_col .. +3, four bytes
// per row packed into one word each (byte k = column jx + lane_col + k).  Three ways to the same bytes, chosen per origin
// (warp-uniform): aligned words and a funnel shift on a word-aligned level, byte loads elsewhere inside the image, and
// reflect-101 addresses for a window that overlaps the border (the values of the reflected border
// cv::buildOpticalFlowPyramid gives the search levels).  Jlane = level image + lane_row * Jpitch; offsets within one level
// image fit 32 bits.
__device__ __forceinline__ void gather_taps(const uint8_t* Jlane, int Jpitch, int lw, int lh, int jx,
                                            int jy, int lane_row, int lane_col, bool packed_ok, unsigned& top, unsigned& bot) {
    using kltsetup::WIN;
    const int x = jx + lane_col;
    if (jx >= 0 && jy >= 0 && jx + WIN < lw && jy + WIN < lh) {
        const int o = jy * Jpitch;
        if (packed_ok) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(Jlane + (o + (x & ~3)));
            const uint32_t* wb = reinterpret_cast<const uint32_t*>(Jlane + (o + Jpitch + (x & ~3)));
            const unsigned sh = (unsigned)(x & 3) * 8u;
            const unsigned t0 = __ldg(w), b0 = __ldg(wb);
            unsigned t1 = 0, b1 = 0;
            if (sh) { t1 = __ldg(w + 1); b1 = __ldg(wb + 1); }   // the next word may lie past the row's end when sh = 0
            top = kltsetup::funnel_r(t0, t1, sh);
            bot = kltsetup::funnel_r(b0, b1, sh);
        } else {
            const uint8_t* q = Jlane + (o + x);
            top = __ldg(q) | (unsigned)__ldg(q + 1) << 8 | (unsigned)__ldg(q + 2) << 16 | (unsigned)__ldg(q + 3) << 24;
            q += Jpitch;
            bot = __ldg(q) | (unsigned)__ldg(q + 1) << 8 | (unsigned)__ldg(q + 2) << 16 | (unsigned)__ldg(q + 3) << 24;
        }
        return;
    }
    const uint8_t* r0 = Jlane + (kltsetup::reflect101_any(jy + lane_row, lh) - lane_row) * Jpitch;
    const uint8_t* r1 = Jlane + (kltsetup::reflect101_any(jy + lane_row + 1, lh) - lane_row) * Jpitch;
    top = 0;
    bot = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xr = kltsetup::reflect101_any(x + k, lw);
        top |= (unsigned)__ldg(r0 + xr) << (8 * k);
        bot |= (unsigned)__ldg(r1 + xr) << (8 * k);
    }
}

// ---- Window layouts.  lk_track runs the level / iteration control flow for both; its Win parameter does a level's window
// work in the warp's shared memory (sN bytes, sD ints) and registers:
//   Win(lane, sN, sD, win)                                 once per track
//   level(Jimg, Jpitch, lw, lh)                            a level's search image
//   setup(Iimg, Ipitch, ix, iy, iw.., A11, A12, A22)      template window and normal matrix (float32, scaled by 2^-20)
//   search(jx, jy)                                         the search pixels of a new integer window origin
//   mismatch(iw.., b1, b2)                                 one iteration's mismatch sums (float32, scaled by 2^-20)
// and gives its kernel instantiation's warps per CTA, launch bounds and per-warp shared memory.
constexpr float LK_SCALE = 1.f / (1 << 20);

// 9 x 9, the window of every shipped configuration.  Lane l < 27 owns the three horizontally adjacent window pixels
// 3l .. 3l+2 (row l / 3, columns 3 (l % 3) ..), so the search-image taps of a lane are 4 consecutive bytes on two rows,
// packed in registers; the integer window sums are order independent.  Lanes 27..31 keep zero taps against a zero
// template, so every lane runs the same straight-line arithmetic.
struct Win9 {
    static constexpr const char* NAME = "fb_klt_kernel";
    static constexpr int WARPS = 8, MIN_CTAS = 32 / WARPS;
    static constexpr int SN_BYTES = kltsetup::SP_BYTES, SD_INTS = kltsetup::SD_INTS;
    __host__ __device__ static constexpr int size(int) { return kltsetup::WIN; }

    const int lane, lane_row, lane_col;
    uint8_t* const sP;
    int* const sD;
    int Jpitch, lw, lh;
    bool packed_ok;   // aliased level 0 may be unaligned
    const uint8_t* Jlane;
    int I0, I1, I2, X0, X1, X2, Y0, Y1, Y2;   // the template values as the iterations use them
    int gsum;                                 // sum |Ix| + |Iy| over the window
    unsigned top, bot;                        // the lane's search taps

    __device__ __forceinline__ Win9(int lane, uint8_t* sN, int* sD, int)
        : lane(lane), lane_row(lane / 3), lane_col(3 * (lane - 3 * (lane / 3))), sP(sN), sD(sD) {}
    __device__ __forceinline__ void level(const uint8_t* Jimg, int pitch, int w, int h) {
        Jpitch = pitch;
        lw = w;
        lh = h;
        packed_ok = ((reinterpret_cast<uintptr_t>(Jimg) | (uintptr_t)Jpitch) & 3) == 0;
        Jlane = Jimg + lane_row * Jpitch;
        top = 0;
        bot = 0;
    }

    // klt_setup.cuh: 12 x 12 neighbourhood -> shared memory (aligned words on the interior path), Scharr at the 10 x 10
    // bilinear footprint, int16 template window (as sign-extended ints) + exact integer normal-equation sums.
    __device__ __forceinline__ void setup(const uint8_t* Iimg, int Ipitch, int ix, int iy, int iw00, int iw01, int iw10,
                                          int iw11, float& A11, float& A12, float& A22) {
        const bool tmpl_aligned = ((reinterpret_cast<uintptr_t>(Iimg) | (uintptr_t)Ipitch) & 3) == 0;
        int Iv[3], Ixv[3], Iyv[3];
        int sA11, sA12, sA22;
        if (tmpl_aligned && kltsetup::patch_interior(ix, iy, lw, lh)) {
            // interior (warp-uniform): interpolate first, differentiate after - same integers, one pass, no derivative patch
            kltsetup::stage_interior(lane, Iimg, Ipitch, lw, ix, iy, sP);
            __syncwarp();
            kltsetup::template_direct(lane, sP, (ix - 1) & 3, iw00, iw01, iw10, iw11, Iv, Ixv, Iyv, sA11, sA12, sA22);
        } else {
            kltsetup::stage_border(lane, Iimg, Ipitch, lw, lh, ix, iy, sP);
            __syncwarp();
            kltsetup::scharr_rows(lane, sP, 0, ix, iy, lw, lh, sD);
            __syncwarp();
            kltsetup::template_rows(lane, sP, 0, sD, iw00, iw01, iw10, iw11, Iv, Ixv, Iyv, sA11, sA12, sA22);
        }
        I0 = Iv[0], I1 = Iv[1], I2 = Iv[2];
        X0 = Ixv[0], X1 = Ixv[1], X2 = Ixv[2];
        Y0 = Iyv[0], Y1 = Iyv[1], Y2 = Iyv[2];
        gsum = __reduce_add_sync(FULL, abs(X0) + abs(X1) + abs(X2) + abs(Y0) + abs(Y1) + abs(Y2));
        // |window sums| <= 81 * 4080^2 = 1.35e9 < 2^31 for the 9 x 9 window: one exact 32-bit redux each
        // (the b sums of the iterations can reach 2.7e9 and keep the split 64-bit reduction)
        A11 = __int2float_rn(__reduce_add_sync(FULL, sA11)) * LK_SCALE;
        A12 = __int2float_rn(__reduce_add_sync(FULL, sA12)) * LK_SCALE;
        A22 = __int2float_rn(__reduce_add_sync(FULL, sA22)) * LK_SCALE;
    }

    __device__ __forceinline__ void search(int jx, int jy) {
        if (lane < 27) gather_taps(Jlane, Jpitch, lw, lh, jx, jy, lane_row, lane_col, packed_ok, top, bot);
    }

    __device__ __forceinline__ void mismatch(int iw00, int iw01, int iw10, int iw11, float& b1, float& b2) const {
        // the 14-bit bilinear weights as signed 16-bit pairs, applied to the packed taps with dp2a (u16 x u8 pairs):
        // the same integers as (J00 iw00 + J01 iw01 + J10 iw10 + J11 iw11 + 2^8) >> 9, exact in int32
        const unsigned W01 = __byte_perm((unsigned)iw00, (unsigned)iw01, 0x5410);
        const unsigned W23 = __byte_perm((unsigned)iw10, (unsigned)iw11, 0x5410);
        const int j0 = kltsetup::dp2a_lo_su16(W01, top, kltsetup::dp2a_lo_su16(W23, bot, 256)) >> 9;
        const int j1 = kltsetup::dp2a_lo_su16(W01, top >> 8, kltsetup::dp2a_lo_su16(W23, bot >> 8, 256)) >> 9;
        const int j2 = kltsetup::dp2a_hi_su16(W01, top, kltsetup::dp2a_hi_su16(W23, bot, 256)) >> 9;
        const int d0 = j0 - I0, d1 = j1 - I1, d2 = j2 - I2;
        const int sb1 = d0 * X0 + d1 * X1 + d2 * X2;
        const int sb2 = d0 * Y0 + d1 * Y1 + d2 * Y2;
        // |b sums| <= max|J - I| * sum|Ix| with |J - I| <= 8160 (both are 8-bit intensities with 5 fractional bits): when
        // 8160 * (sum|Ix| + sum|Iy|) < 2^31 the mismatch sums fit one exact 32-bit redux each (true for every window whose
        // mean |gradient| is below ~3200 of the possible 8160, i.e. anything but a synthetic checkerboard;
        // 8162 * 262000 < 2^31); otherwise the split 64-bit reduction is kept.  Same integers either way.
        if (gsum < 262000) {
            b1 = __int2float_rn(__reduce_add_sync(FULL, sb1)) * LK_SCALE;
            b2 = __int2float_rn(__reduce_add_sync(FULL, sb2)) * LK_SCALE;
        } else {
            b1 = __ll2float_rn(warp_sum64(sb1)) * LK_SCALE;
            b2 = __ll2float_rn(warp_sum64(sb2)) * LK_SCALE;
        }
    }
};

// Any window from 3 to 31 but 9.  Lane c owns window column c (klt_setup.cuh, win_*): the level set-up stages the
// (win + 3)^2 template neighbourhood, its Scharr derivatives and the template into the warp's shared memory, and each
// move of the integer search origin stages the (win + 1)^2 search bytes into the neighbourhood's buffer.  A lane's column
// sums are exact in int32, the window sums in 64 bits.  Per warp: the staged bytes (WN_BYTES), then the derivative plane,
// the template derivatives (ints) and the template intensities (shorts) in one int array; 11 272 bytes.
struct WinAny {
    static constexpr const char* NAME = "fb_klt_win_kernel";
    static constexpr int WARPS = 4, MIN_CTAS = 0;
    static constexpr int SN_BYTES = kltsetup::WN_BYTES;
    static constexpr int SD_INTS = kltsetup::WD_INTS + kltsetup::WT_ELEMS + kltsetup::WT_ELEMS / 2;
    __host__ __device__ static constexpr int size(int win) { return win; }

    const int lane, win;
    uint8_t* const sN;
    int* const sD;
    int* const sG;
    short* const sI;
    const uint8_t* Jimg;
    int Jpitch, lw, lh;

    __device__ __forceinline__ WinAny(int lane, uint8_t* sN, int* sD, int win)
        : lane(lane), win(win), sN(sN), sD(sD), sG(sD + kltsetup::WD_INTS),
          sI(reinterpret_cast<short*>(sD + kltsetup::WD_INTS + kltsetup::WT_ELEMS)) {}
    __device__ __forceinline__ void level(const uint8_t* img, int pitch, int w, int h) {
        Jimg = img;
        Jpitch = pitch;
        lw = w;
        lh = h;
    }

    __device__ __forceinline__ void setup(const uint8_t* Iimg, int Ipitch, int ix, int iy, int iw00, int iw01, int iw10,
                                          int iw11, float& A11, float& A12, float& A22) {
        kltsetup::win_stage(lane, Iimg, Ipitch, lw, lh, ix - 1, iy - 1, win + 3, sN);
        __syncwarp();
        kltsetup::win_scharr(lane, sN, ix, iy, lw, lh, win, sD);
        __syncwarp();
        int sA11, sA12, sA22;
        kltsetup::win_template(lane, sN, sD, win, iw00, iw01, iw10, iw11, sI, sG, sA11, sA12, sA22);
        A11 = __ll2float_rn(warp_sum64(sA11)) * LK_SCALE;
        A12 = __ll2float_rn(warp_sum64(sA12)) * LK_SCALE;
        A22 = __ll2float_rn(warp_sum64(sA22)) * LK_SCALE;
    }

    __device__ __forceinline__ void search(int jx, int jy) {
        __syncwarp();            // the template phase or the previous iteration is done with sN
        kltsetup::win_stage(lane, Jimg, Jpitch, lw, lh, jx, jy, win + 1, sN);
        __syncwarp();
    }

    __device__ __forceinline__ void mismatch(int iw00, int iw01, int iw10, int iw11, float& b1, float& b2) const {
        int sb1, sb2;
        kltsetup::win_mismatch(lane, sN, sI, sG, win, iw00, iw01, iw10, iw11, sb1, sb2);
        b1 = __ll2float_rn(warp_sum64(sb1)) * LK_SCALE;
        b2 = __ll2float_rn(warp_sum64(sb2)) * LK_SCALE;
    }
};

// One calcOpticalFlowPyrLK track for one point with Win's window (whole warp cooperates).
// Ipyr = template pyramid, Jpyr = search pyramid.  nxt: in = initial guess, out = result.
// COUNT (measurement instantiation): work gains 1 << 16 per level set-up that builds the template and 1 per iteration that
// forms the mismatch sums (one register for both: the product instantiation has none to spare).
template <bool COUNT, class Win>
__device__ bool lk_track(const PyrView& Ipyr, const PyrView& Jpyr, int frame, float2 pt, float2& nxt, int maxlevel, int win,
                         int max_iter, double eps2, float eps_lo, float eps_hi, float eig_q, float& err_out, uint8_t* sN, int* sD,
                         int lane, int& work) {
    win = Win::size(win);
    Win W(lane, sN, sD, win);
    const float half = (win - 1) * 0.5f;
    bool status = true;
    float err = 0.f;   // the numerator q of minEig (lk_eig_num)

    for (int level = maxlevel; level >= 0; --level) {
        const int lw = Ipyr.w[level], lh = Ipyr.h[level];
        const uint8_t* Iimg = Ipyr.lvl[level] + Ipyr.fstride[level] * frame;
        const uint8_t* Jimg = Jpyr.lvl[level] + Jpyr.fstride[level] * frame;
        const int Ipitch = Ipyr.pitch[level], Jpitch = Jpyr.pitch[level];
        W.level(Jimg, Jpitch, lw, lh);
        const float sc = __int_as_float((127 - level) << 23);   // 2^-level, exactly 1.f / (1 << level)
        float2 prevPt = make_float2(pt.x * sc, pt.y * sc);
        float2 nextPt;
        if (level == maxlevel) nextPt = make_float2(nxt.x * sc, nxt.y * sc);
        else nextPt = make_float2(nxt.x * 2.f, nxt.y * 2.f);
        nxt = nextPt;
        prevPt.x -= half;
        prevPt.y -= half;
        const int ix = __float2int_rd(prevPt.x), iy = __float2int_rd(prevPt.y);
        if (ix < -win || ix >= lw || iy < -win || iy >= lh) {
            if (level == 0) { status = false; err = 0.f; }
            continue;
        }
        if (COUNT) work += 1 << 16;
        float a = prevPt.x - (float)ix, b = prevPt.y - (float)iy;
        int iw00, iw01, iw10, iw11;
        LK_WEIGHTS(a, b, iw00, iw01, iw10, iw11);
        __syncwarp();                    // the previous level's iterations are done with the warp's shared memory
        float A11, A12, A22;
        W.setup(Iimg, Ipitch, ix, iy, iw00, iw01, iw10, iw11, A11, A12, A22);
        float D = A11 * A22 - A12 * A12;
        err = lk_eig_num(A11, A12, A22);
        if (err < eig_q || D < LK_MIN_DET) {
            if (level == 0) status = false;
            continue;
        }
        D = 1.f / D;
        nextPt.x -= half;
        nextPt.y -= half;
        float2 prevDelta = make_float2(0.f, 0.f);
        // The search pixels are fetched when the integer origin (jx, jy) of the window moves and kept while it does not
        // (sub-pixel steps only change the bilinear weights).  nxt is written where the loop ends, not every iteration:
        // the values are those OpenCV leaves in nextPts at each exit.
        int cjx = INT_MIN, cjy = INT_MIN;
        int j = 0;
        for (; j < max_iter; ++j) {
            const int jx = __float2int_rd(nextPt.x), jy = __float2int_rd(nextPt.y);
            if ((jx != cjx) | (jy != cjy)) {
                if (jx < -win || jx >= lw || jy < -win || jy >= lh) {
                    if (j > 0) nxt = make_float2(nextPt.x + half, nextPt.y + half);
                    if (level == 0) status = false;
                    break;
                }
                W.search(jx, jy);
                cjx = jx;
                cjy = jy;
            }
            if (COUNT) ++work;
            a = nextPt.x - (float)jx;
            b = nextPt.y - (float)jy;
            LK_WEIGHTS(a, b, iw00, iw01, iw10, iw11);
            float b1, b2;
            W.mismatch(iw00, iw01, iw10, iw11, b1, b2);
            const float2 delta = lk_step(A11, A12, A22, D, b1, b2);
            nextPt.x += delta.x;
            nextPt.y += delta.y;
            LK_CONVERGED(conv, delta, eps2, eps_lo, eps_hi);
            if (conv) {
                nxt = make_float2(nextPt.x + half, nextPt.y + half);
                break;
            }
            if (j > 0 && LK_OSCILLATES(delta, prevDelta)) {
                nxt = make_float2((nextPt.x + half) - delta.x * 0.5f, (nextPt.y + half) - delta.y * 0.5f);
                break;
            }
            prevDelta = delta;
        }
        if (j == max_iter && j > 0) nxt = make_float2(nextPt.x + half, nextPt.y + half);
    }
    err_out = err;
    return status;
}

// One keypoint, whole warp: forward track, checks, backward track, forward-backward test (feature_tracker.cpp:35-137).
// counts (measurement instantiation): level set-ups and iterations of both tracks, at 2 i and 2 i + 1.
template <bool COUNT, class Win>
__device__ __forceinline__ void klt_one(const KltArgs& A, int i, uint8_t* sNw, int* sDw, int lane, int32_t* counts, int win) {
    const int frame = A.frame_idx ? A.frame_idx[i] : A.first_frame + i / A.per_frame;
    int maxlevel = A.lvls ? (int)A.lvls[i] : A.lvl_all;
    if (maxlevel > A.prev.nlev - 1) maxlevel = A.prev.nlev - 1;  // feature_tracker.cpp:50-52
    if (maxlevel < 0) maxlevel = 0;
    const float2 kp = A.kps[i];
    float2 fwd = A.priors[i];
    float err = 0.f;
    int work = 0;
    // x < 0 marks an empty slot of a fixed-stride batch (the detectors pad their output with (-1, -1),
    // ov2_describe uses the same rule): status 0, prior untouched, no work
    bool ok = kp.x >= 0.f && lk_track<COUNT, Win>(A.prev, A.cur, frame, kp, fwd, maxlevel, win, A.max_iter, A.eps2, A.eps_lo,
                                                  A.eps_hi, A.eig_q, err, sNw, sDw, lane, work);
    // feature_tracker.cpp:79-101 (err > ferr and the distance test through the thresholds of KltArgs)
    if (ok && err > A.ferr_q) ok = false;
    if (ok) {
        const float w0 = (float)A.cur.w[0], h0 = (float)A.cur.h[0];
        if (!(1.f <= fwd.x && fwd.x < w0 - 1.f && 1.f <= fwd.y && fwd.y < h0 - 1.f)) ok = false;
    }
    if (ok) {
        // backward: template from the current image at the forward result, search the previous image
        float2 back = kp;
        float err2 = 0.f;
        const bool ok2 = lk_track<COUNT, Win>(A.cur, A.prev, frame, fwd, back, 0, win, A.max_iter, A.eps2, A.eps_lo, A.eps_hi,
                                              A.eig_q, err2, sNw, sDw, lane, work);
        if (!ok2) ok = false;
        else {
            float dx = kp.x - back.x, dy = kp.y - back.y;
            if ((double)dx * (double)dx + (double)dy * (double)dy > A.fb_s) ok = false;
        }
    }
    if (lane == 0) {
        A.priors[i] = fwd;
        A.status[i] = ok ? 1 : 0;
        if (COUNT) {
            counts[2 * i] = work >> 16;
            counts[2 * i + 1] = work & 0xFFFF;
        }
    }
}

// Keypoints need very different iteration counts (1 .. 30 per level), so a static warp <-> keypoint
// assignment leaves SM slots idle while the slowest warp of a CTA finishes.  When the grid exceeds the
// resident CTAs, the launch fills the GPU once and every warp pulls the next keypoint from a global counter;
// it asks for the next index before tracking the current one, so the atomic's round trip overlaps the track.
template <bool COUNT, class Win>
__global__ void __launch_bounds__(Win::WARPS * 32, Win::MIN_CTAS) fb_klt_kernel(KltArgs A, int32_t* counts, int win) {
    __shared__ __align__(16) uint8_t sNall[Win::WARPS][Win::SN_BYTES];
    __shared__ __align__(16) int sDall[Win::WARPS][Win::SD_INTS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int i = blockIdx.x * Win::WARPS + warp;
    if (A.work_counter) {
        int first = 0;
        if (lane == 0) first = atomicAdd(A.work_counter, 1);
        i = __shfl_sync(FULL, first, 0);
    }
    while (i < A.n) {
        int nxt_i = 0;
        if (A.work_counter && lane == 0) nxt_i = atomicAdd(A.work_counter, 1);
        klt_one<COUNT, Win>(A, i, sNall[warp], sDall[warp], lane, counts, win);
        if (!A.work_counter) return;
        i = __shfl_sync(FULL, nxt_i, 0);
    }
}

// Depth cv::buildOpticalFlowPyramid(img, pyr, Size(win, win), maxlevel) reaches: it stops before a level whose width or
// height would be <= win.  calcOpticalFlowPyrLK tracks from there, and the reference clamps nbpyrlvl to it
// (feature_tracker.cpp:50-52), so on small images the tracker starts at a shallower level than the pyramid holds.
int optflow_levels(const ov2_pyr* p, int win, int maxlevel) {
    for (int l = 0; l < maxlevel; ++l)
        if (p->w[l + 1] <= win || p->h[l + 1] <= win) return l;
    return maxlevel;
}

// Launches fb_klt_kernel with Win's layout, the counting instantiation when d_counts is set: one warp per keypoint, or the
// persistent launch over the work counter when the grid exceeds the resident CTAs.
template <class Win>
ov2_status klt_run(ov2_ctx* ctx, KltArgs& A, int n, int32_t* d_counts, int win) {
    constexpr int threads = Win::WARPS * 32;
    int grid = div_up(n, Win::WARPS), per_sm = 0;
    A.work_counter = nullptr;
    OV2_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fb_klt_kernel<false, Win>, threads, 0));
    const int resident = per_sm * ctx->sm_count;
    if (grid > resident) {
        const ov2_status st = ov2_scratch(ctx, 1, A.work_counter);
        if (st != OV2_OK) return st;
        OV2_CUDA(ctx, cudaMemsetAsync(A.work_counter, 0, sizeof(int), ctx->stream));
        grid = resident;
    }
    if (d_counts)
        OV2_LAUNCH(ctx, Win::NAME, (fb_klt_kernel<true, Win><<<grid, threads, 0, ctx->stream>>>(A, d_counts, win)));
    else
        OV2_LAUNCH(ctx, Win::NAME, (fb_klt_kernel<false, Win><<<grid, threads, 0, ctx->stream>>>(A, nullptr, win)));
    return OV2_OK;
}

// ov2_fb_klt, and with counts_out the counting instantiation of the kernel behind ov2_debug_klt_counts
ov2_status klt_launch(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int n,
                      const int32_t* frame_idx, int first_frame, int per_frame, const uint8_t* nbpyrlvl, int nbpyrlvl_all,
                      const float* kps, float* priors_inout, uint8_t* status_out, int32_t* counts_out) {
    if (!ctx || !prev || !cur || !prm || n < 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_fb_klt: bad arguments");
    if (n == 0) return OV2_OK;  // feature_tracker.cpp:43-46
    if (!kps || !priors_inout || !status_out || (!frame_idx && per_frame <= 0))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_fb_klt: null array");
    if (prm->win < 3 || prm->win > kltsetup::WMAX)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_fb_klt: nwinsize must be 3 .. 31");
    if (!ov2_pyr_pair_ok(prev, cur)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_fb_klt: pyramids not built / mismatched");
    if (!frame_idx && (first_frame < 0 || first_frame + (n + per_frame - 1) / per_frame > prev->batch))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_fb_klt: more frames than pyramid slots");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    KltArgs A;
    A.prev = make_view(prev);
    A.cur = make_view(cur);
    // every depth clamp of the kernels reads prev.nlev
    A.prev.nlev = A.cur.nlev = optflow_levels(prev, prm->win, A.prev.nlev - 1) + 1;
    A.n = n;
    A.first_frame = first_frame;
    A.per_frame = per_frame;
    A.lvl_all = nbpyrlvl_all;
    A.max_iter = prm->max_iter;
    A.eps2 = (double)prm->eps * (double)prm->eps;
    A.eps_lo = (float)(A.eps2 * (1.0 - 1e-6));
    A.eps_hi = (float)(A.eps2 * (1.0 + 1e-6));
    A.eig_q = kltsetup::klt_eig_q(prm->win, LK_MIN_EIG);
    A.ferr_q = kltsetup::klt_ferr_q(prm->win, prm->ferr);
    A.fb_s = kltsetup::klt_fb_s(prm->fb_dist);
    if ((st = ov2_stage_in(ctx, frame_idx, (size_t)n, A.frame_idx)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, nbpyrlvl, (size_t)n, A.lvls)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, kps, (size_t)n, A.kps)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, priors_inout, (size_t)n, A.priors, true)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, status_out, (size_t)n, A.status)) != OV2_OK) return st;
    int32_t* d_counts = nullptr;
    if (counts_out && (st = ov2_stage_out(ctx, counts_out, 2 * (size_t)n, d_counts)) != OV2_OK) return st;
    // 9 x 9 (every shipped configuration) keeps its own layout; every other size runs the general one
    st = prm->win == 9 ? klt_run<Win9>(ctx, A, n, d_counts, prm->win) : klt_run<WinAny>(ctx, A, n, d_counts, prm->win);
    if (st != OV2_OK) return st;
    return ov2_end(ctx);
}

}  // namespace

extern "C" ov2_status ov2_fb_klt(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm,
                                 int n, const int32_t* frame_idx, int first_frame, int per_frame, const uint8_t* nbpyrlvl,
                                 int nbpyrlvl_all, const float* kps, float* priors_inout, uint8_t* status_out) {
    return klt_launch(ctx, prev, cur, prm, n, frame_idx, first_frame, per_frame, nbpyrlvl, nbpyrlvl_all, kps, priors_inout,
                      status_out, nullptr);
}

// Measurement hook: ov2_fb_klt with the same arguments and results, plus the work each keypoint took: counts_out[2 i] level
// set-ups (template built) and counts_out[2 i + 1] iterations (mismatch sums formed), forward and backward tracks together.
// A second instantiation of the kernel: the product launch carries no counter.
extern "C" ov2_status ov2_debug_klt_counts(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm,
                                           int n, const int32_t* frame_idx, int first_frame, int per_frame,
                                           const uint8_t* nbpyrlvl, int nbpyrlvl_all, const float* kps, float* priors_inout,
                                           uint8_t* status_out, int32_t* counts_out) {
    if (!counts_out && n > 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_debug_klt_counts: null counts array");
    return klt_launch(ctx, prev, cur, prm, n, frame_idx, first_frame, per_frame, nbpyrlvl, nbpyrlvl_all, kps, priors_inout,
                      status_out, counts_out);
}
