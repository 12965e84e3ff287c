// K (level set-up): template patch staging, Scharr derivatives and the int16 template / derivative
// window of one Lucas-Kanade level, for the 9 x 9 window (all reference configurations,
// /root/reference/src/feature_tracker.cpp:35-137 via cv::calcOpticalFlowPyrLK), and the reflect-101 /
// dp2a / funnel-shift helpers that the tracker's iterations (frontend_klt.cu) use as well.  The win_* functions at the
// end are the same phases for every other window size from 3 to 31 (fb_klt_win_kernel), checked lane by lane in
// tests/test_klt_win_lane_code.py.
//
// Written as plain per-lane functions (no warp intrinsics; the phases are separated by __syncwarp in
// the kernel) so that tests/test_host_logic.py can compile the SAME code for the host and check it
// against the definition, lane by lane (test_klt_level_setup_lane_code_matches_definition, and
// tests/test_klt_setup_host.py for the split staging and the int-output template functions the kernel calls).
//
// Shared-memory layout per warp:
//   sP  : 12 rows x 16 bytes.  Row r holds image row iy-1+r; byte (r, c) of the 12 x 12 neighbourhood
//         (c = 0 is image column ix-1) lives at sP[r * 16 + off + c], off = (ix-1) & 3 on the word-aligned
//         interior path (rows are staged as 4 ALIGNED 32-bit words each), off = 0 on the border path.
//   sD  : 10 rows x 12 ints, (dx & 0xFFFF) | (dy << 16) of the Scharr derivative at image position
//         (iy + r, ix + c); 0 outside the image (cv::buildOpticalFlowPyramid's BORDER_CONSTANT planes).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define KLT_HD __host__ __device__ __forceinline__
#else
#define KLT_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define KLT_LDG8(p) __ldg(p)
#define KLT_LDG32(p) __ldg(p)
#else
#define KLT_LDG8(p) (*(p))
#define KLT_LDG32(p) (*(p))
#endif

namespace kltsetup {

constexpr int WIN = 9;
constexpr int PW = WIN + 3;      // 12: u8 neighbourhood
constexpr int DW = WIN + 1;      // 10: derivative patch
constexpr int SP_PITCH = 16;     // bytes
constexpr int SD_PITCH = 12;     // ints
constexpr int SP_BYTES = PW * SP_PITCH;   // 192
constexpr int SD_INTS = DW * SD_PITCH;    // 120

KLT_HD int reflect101_any(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * (n - 1) - i;
    }
    return i;
}

// true when the whole 12 x 12 neighbourhood (and therefore every Scharr tap) lies inside the image
KLT_HD bool patch_interior(int ix, int iy, int lw, int lh) { return ix >= 1 && iy >= 1 && ix + PW - 1 <= lw && iy + PW - 1 <= lh; }

// Phase 1, interior path (aligned image, patch_interior()): the 12 rows as 4 aligned words each, off = (ix - 1) & 3.  Word i
// of sP is staged by lane i & 31: lane l holds row l >> 2 and, for l < 16, row 8 + (l >> 2), both at word l & 3 of the row.
// Offsets within one level image fit 32 bits (as in the search gathers), so the lane forms one 32-bit offset from the level's
// base and reaches its second row 8 pitches further.
KLT_HD void stage_interior(int lane, const uint8_t* img, int pitch, int lw, int ix, int iy, uint8_t* sP) {
    const int xw = ((ix - 1) & ~3) + 4 * (lane & 3);   // the lane's word column (>= 0), word aligned
    uint32_t* sPw = reinterpret_cast<uint32_t*>(sP);
    // a word starting at or beyond lw holds no byte the patch needs (and may lie outside the buffer)
    unsigned w0 = 0u, w1 = 0u;
    if (xw < lw) {
        const uint8_t* p = img + ((iy - 1 + (lane >> 2)) * pitch + xw);
        w0 = KLT_LDG32(reinterpret_cast<const uint32_t*>(p));
        if (lane < 16) w1 = KLT_LDG32(reinterpret_cast<const uint32_t*>(p + 8 * pitch));
    }
    sPw[lane] = w0;
    if (lane < 16) sPw[lane + 32] = w1;
}

// Phase 1, border path: the 12 x 12 neighbourhood byte by byte through reflect-101, off = 0.
KLT_HD void stage_border(int lane, const uint8_t* img, int pitch, int lw, int lh, int ix, int iy, uint8_t* sP) {
    for (int i = lane; i < PW * PW; i += 32) {
        const int r = i / PW, c = i - r * PW;
        const int y = reflect101_any(iy - 1 + r, lh), x = reflect101_any(ix - 1 + c, lw);
        sP[r * SP_PITCH + c] = KLT_LDG8(img + (size_t)y * pitch + x);
    }
}

// Phase 1 (all lanes), either path.  Returns off.  `aligned`: image base and pitch are multiples of 4.
KLT_HD int stage_patch(int lane, const uint8_t* img, int pitch, int lw, int lh, int ix, int iy, bool aligned, uint8_t* sP) {
    if (aligned && patch_interior(ix, iy, lw, lh)) {
        stage_interior(lane, img, pitch, lw, ix, iy, sP);
        return (ix - 1) & 3;
    }
    stage_border(lane, img, pitch, lw, lh, ix, iy, sP);
    return 0;
}

// Phase 2 (all lanes): Scharr.  Lane l < 30 owns derivative row l / 3, columns 4 (l % 3) .. +3 (the
// last group has 2 columns): 3 x 6 byte loads, the vertical [3 10 3] / [-1 0 1] passes once per column.
KLT_HD void scharr_rows(int lane, const uint8_t* sP, int off, int ix, int iy, int lw, int lh, int* sD) {
    if (lane >= 30) return;
    const int r = lane / 3, g = lane - 3 * r;
    const int c0 = 4 * g, nout = g == 2 ? 2 : 4;
    const uint8_t* p0 = sP + r * SP_PITCH + off + c0;   // neighbourhood row r (image row iy-1+r), column c0
    int vs[6], vd[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        if (j < nout + 2) {
            const int a = p0[j], b = p0[SP_PITCH + j], c = p0[2 * SP_PITCH + j];
            vs[j] = (a + c) * 3 + b * 10;
            vd[j] = c - a;
        } else {
            vs[j] = 0; vd[j] = 0;
        }
    }
    const int y = iy + r;
    const bool yin = y >= 0 && y < lh;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j < nout) {
            const int x = ix + c0 + j;
            int dx = 0, dy = 0;
            if (yin && x >= 0 && x < lw) {
                dx = vs[j + 2] - vs[j];
                dy = (vd[j] + vd[j + 2]) * 3 + vd[j + 1] * 10;
            }
            sD[r * SD_PITCH + c0 + j] = (int)(((unsigned)dx & 0xFFFFu) | ((unsigned)dy << 16));
        }
    }
}

// Phase 3 (lanes 0..26; others get zeros): window pixels 3l .. 3l+2 = row l / 3, columns 3 (l % 3) .. +2.
// OpenCV's fixed point: I = (bilinear(u8) * 2^14 + 2^8) >> 9, Ix / Iy = (bilinear(s16) + 2^13) >> 14.
// OpenCV stores the results as int16; they fit it (0 <= I <= 8160, |Ix|, |Iy| <= 4081 even with iw11 = -1), so the int
// outputs are the int16 values already sign-extended, as the iterations use them.
KLT_HD void template_rows(int lane, const uint8_t* sP, int off, const int* sD, int iw00, int iw01, int iw10, int iw11,
                          int* Iv, int* Ixv, int* Iyv, int& sA11, int& sA12, int& sA22) {
    sA11 = 0; sA12 = 0; sA22 = 0;
    Iv[0] = Iv[1] = Iv[2] = 0; Ixv[0] = Ixv[1] = Ixv[2] = 0; Iyv[0] = Iyv[1] = Iyv[2] = 0;
    if (lane >= 27) return;
    const int y = lane / 3, x0 = 3 * (lane - 3 * y);
    const uint8_t* q = sP + (y + 1) * SP_PITCH + off + x0 + 1;
    int t[4], b[4], dxt[4], dyt[4], dxb[4], dyb[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        t[j] = q[j];
        b[j] = q[SP_PITCH + j];
        const int d0 = sD[y * SD_PITCH + x0 + j], d1 = sD[(y + 1) * SD_PITCH + x0 + j];
        dxt[j] = (int)(short)(d0 & 0xFFFF); dyt[j] = d0 >> 16;
        dxb[j] = (int)(short)(d1 & 0xFFFF); dyb[j] = d1 >> 16;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int ival = (t[k] * iw00 + t[k + 1] * iw01 + b[k] * iw10 + b[k + 1] * iw11 + (1 << 8)) >> 9;
        const int ixval = (dxt[k] * iw00 + dxt[k + 1] * iw01 + dxb[k] * iw10 + dxb[k + 1] * iw11 + (1 << 13)) >> 14;
        const int iyval = (dyt[k] * iw00 + dyt[k + 1] * iw01 + dyb[k] * iw10 + dyb[k + 1] * iw11 + (1 << 13)) >> 14;
        Iv[k] = ival; Ixv[k] = ixval; Iyv[k] = iyval;
        sA11 += ixval * ixval;
        sA12 += ixval * iyval;
        sA22 += iyval * iyval;
    }
}
KLT_HD void template_rows(int lane, const uint8_t* sP, int off, const int* sD, int iw00, int iw01, int iw10, int iw11,
                          short* Iv, short* Ixv, short* Iyv, int& sA11, int& sA12, int& sA22) {
    int v[3], x[3], y[3];
    template_rows(lane, sP, off, sD, iw00, iw01, iw10, iw11, v, x, y, sA11, sA12, sA22);
    for (int k = 0; k < 3; ++k) { Iv[k] = (short)v[k]; Ixv[k] = (short)x[k]; Iyv[k] = (short)y[k]; }
}

// dp2a: signed 16-bit halves of a (bilinear weights: iw11 = 16384 - others can round to -1) times UNSIGNED bytes of b
// (pixels; lo: bytes 0, 1; hi: bytes 2, 3), plus c
KLT_HD int dp2a_lo_su16(unsigned a, unsigned b, int c) {
#if defined(__CUDA_ARCH__)
    int d;
    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#else
    return c + (int)(short)(a & 0xFFFFu) * (int)(b & 255u) + (int)(short)(a >> 16) * (int)((b >> 8) & 255u);
#endif
}
KLT_HD int dp2a_hi_su16(unsigned a, unsigned b, int c) {
#if defined(__CUDA_ARCH__)
    int d;
    asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#else
    return c + (int)(short)(a & 0xFFFFu) * (int)((b >> 16) & 255u) + (int)(short)(a >> 16) * (int)(b >> 24);
#endif
}
KLT_HD unsigned funnel_r(unsigned lo, unsigned hi, unsigned sh) {   // bytes of hi:lo shifted right by sh bits (sh = 0, 8, 16, 24)
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
}

// Phases 2 + 3 in one for the INTERIOR case (patch_interior(): every Scharr tap is a real pixel, no reflected border and
// no zero plane).  The bilinear interpolation and the Scharr filter are both exact integer linear maps, so they commute:
//   bilinear(Scharr(P))  ==  Scharr(W),   W[r][c] = P[r][c] iw00 + P[r][c+1] iw01 + P[r+1][c] iw10 + P[r+1][c+1] iw11
// with W <= 255 * 16385 (22 bits) and the Scharr sums of W below 2^27: same integers as template_rows() produces from the
// int16 derivative planes, then the same roundings (I: (W + 2^8) >> 9, Ix / Iy: (. + 2^13) >> 14).  A lane forms the 3 x 5 W
// values around its three pixels straight from the staged bytes with dp2a; nothing is written to sD and no second
// __syncwarp is needed.  Lane l < 27 owns window pixels (l / 3, 3 (l % 3) ..+2) as in template_rows(), int outputs as there.
KLT_HD void template_direct(int lane, const uint8_t* sP, int off, int iw00, int iw01, int iw10, int iw11,
                            int* Iv, int* Ixv, int* Iyv, int& sA11, int& sA12, int& sA22) {
    sA11 = 0; sA12 = 0; sA22 = 0;
    Iv[0] = Iv[1] = Iv[2] = 0; Ixv[0] = Ixv[1] = Ixv[2] = 0; Iyv[0] = Iyv[1] = Iyv[2] = 0;
    if (lane >= 27) return;
    const int y = lane / 3, x0 = 3 * (lane - 3 * y);
    const unsigned W01 = ((unsigned)iw00 & 0xFFFFu) | ((unsigned)iw01 << 16);
    const unsigned W23 = ((unsigned)iw10 & 0xFFFFu) | ((unsigned)iw11 << 16);
    // neighbourhood rows y .. y+3, bytes bo .. bo+5 of each 16-byte row (bo = off + x0 <= 9)
    const int bo = off + x0, wi = bo >> 2;
    const unsigned sh = (unsigned)(bo & 3) * 8u;
    unsigned lo[4], hi[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const uint32_t* rw = reinterpret_cast<const uint32_t*>(sP + (y + r) * SP_PITCH);
        const unsigned w0 = rw[wi], w1 = rw[wi + 1], w2 = wi < 2 ? rw[wi + 2] : 0u;
        lo[r] = funnel_r(w0, w1, sh);      // bytes bo .. bo+3
        hi[r] = funnel_r(w1, w2, sh);      // bytes bo+4 .. bo+7 (only bo+4, bo+5 are used)
    }
    int W[3][5];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const unsigned t = lo[r], b = lo[r + 1];
        const unsigned t3 = funnel_r(lo[r], hi[r], 24u), b3 = funnel_r(lo[r + 1], hi[r + 1], 24u);
        W[r][0] = dp2a_lo_su16(W01, t, dp2a_lo_su16(W23, b, 0));
        W[r][1] = dp2a_lo_su16(W01, t >> 8, dp2a_lo_su16(W23, b >> 8, 0));
        W[r][2] = dp2a_hi_su16(W01, t, dp2a_hi_su16(W23, b, 0));
        W[r][3] = dp2a_lo_su16(W01, t3, dp2a_lo_su16(W23, b3, 0));
        W[r][4] = dp2a_lo_su16(W01, hi[r], dp2a_lo_su16(W23, hi[r + 1], 0));
    }
    int vs[5], vd[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        vs[c] = (W[0][c] + W[2][c]) * 3 + W[1][c] * 10;
        vd[c] = W[2][c] - W[0][c];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int ival = (W[1][k + 1] + (1 << 8)) >> 9;
        const int ixval = (vs[k + 2] - vs[k] + (1 << 13)) >> 14;
        const int iyval = ((vd[k] + vd[k + 2]) * 3 + vd[k + 1] * 10 + (1 << 13)) >> 14;
        Iv[k] = ival; Ixv[k] = ixval; Iyv[k] = iyval;
        sA11 += ixval * ixval;
        sA12 += ixval * iyval;
        sA22 += iyval * iyval;
    }
}
KLT_HD void template_direct(int lane, const uint8_t* sP, int off, int iw00, int iw01, int iw10, int iw11,
                            short* Iv, short* Ixv, short* Iyv, int& sA11, int& sA12, int& sA22) {
    int v[3], x[3], y[3];
    template_direct(lane, sP, off, iw00, iw01, iw10, iw11, v, x, y, sA11, sA12, sA22);
    for (int k = 0; k < 3; ++k) { Iv[k] = (short)v[k]; Ixv[k] = (short)x[k]; Iyv[k] = (short)y[k]; }
}

// ---- Any window from 3 to 31 (fb_klt_win_kernel): lane c owns window column c, every row of it.
//
// Shared-memory layout per warp (win <= WMAX):
//   sN  : (n rows) x WN_PITCH bytes, byte (r, c) = image (reflect101(y0 + r), reflect101(x0 + c)); the template level
//         set-up stages the (win + 3)^2 neighbourhood from (ix - 1, iy - 1), the iterations the (win + 1)^2 search bytes
//         from (jx, jy) into the same buffer.
//   sD  : (win + 1) rows x WG_PITCH ints, Scharr (dx & 0xFFFF) | (dy << 16) at image (iy + r, ix + c); 0 outside the image.
//   sI  : win rows x WG_PITCH shorts, the template intensities (5 fractional bits).
//   sG  : win rows x WG_PITCH ints, the template derivatives (Ix & 0xFFFF) | (Iy << 16).
// Per lane, |Ix|, |Iy| <= 4080 and |J - I| <= 8160, so 31 rows keep every per-lane sum below 2^31.
constexpr int WMAX = 31;
constexpr int WN_PITCH = 36;                       // bytes: the neighbourhood is at most 34 wide
constexpr int WN_BYTES = (WMAX + 3) * WN_PITCH;    // 1224
constexpr int WG_PITCH = 32;                       // elements of a derivative / template row
constexpr int WD_INTS = (WMAX + 1) * WG_PITCH;     // 1024
constexpr int WT_ELEMS = WMAX * WG_PITCH;          // 992

// n x n bytes from origin (x0, y0), reflect-101 outside the image; lanes stride the columns (n <= 34).
KLT_HD void win_stage(int lane, const uint8_t* img, int pitch, int lw, int lh, int x0, int y0, int n, uint8_t* sN) {
    const bool inside = x0 >= 0 && y0 >= 0 && x0 + n <= lw && y0 + n <= lh;
    for (int r = 0; r < n; ++r) {
        const uint8_t* row = img + (size_t)(inside ? y0 + r : reflect101_any(y0 + r, lh)) * pitch;
        for (int c = lane; c < n; c += 32) sN[r * WN_PITCH + c] = KLT_LDG8(row + (inside ? x0 + c : reflect101_any(x0 + c, lw)));
    }
}

// Scharr of the staged (win + 3)^2 neighbourhood: lane c <= win fills derivative column c, rows 0 .. win, rolling the
// three neighbourhood rows it reads down the column.
KLT_HD void win_scharr(int lane, const uint8_t* sN, int ix, int iy, int lw, int lh, int win, int* sD) {
    if (lane > win) return;
    const int c = lane;
    const bool xin = ix + c >= 0 && ix + c < lw;
    const uint8_t* p = sN + c;
    int a0 = p[0], a1 = p[1], a2 = p[2];
    int b0 = p[WN_PITCH], b1 = p[WN_PITCH + 1], b2 = p[WN_PITCH + 2];
    for (int r = 0; r <= win; ++r) {
        const uint8_t* q = p + (r + 2) * WN_PITCH;
        const int c0 = q[0], c1 = q[1], c2 = q[2];
        const int y = iy + r;
        int dx = 0, dy = 0;
        if (xin && y >= 0 && y < lh) {
            dx = ((a2 + c2) * 3 + b2 * 10) - ((a0 + c0) * 3 + b0 * 10);
            dy = ((c0 - a0) + (c2 - a2)) * 3 + (c1 - a1) * 10;
        }
        sD[r * WG_PITCH + c] = (int)(((unsigned)dx & 0xFFFFu) | ((unsigned)dy << 16));
        a0 = b0; a1 = b1; a2 = b2;
        b0 = c0; b1 = c1; b2 = c2;
    }
}

// The template window: lane c < win fills column c of sI / sG and returns its share of the normal-equation sums
// (zeros for lanes >= win).  OpenCV's fixed point as in template_rows().
KLT_HD void win_template(int lane, const uint8_t* sN, const int* sD, int win, int iw00, int iw01, int iw10, int iw11,
                         short* sI, int* sG, int& sA11, int& sA12, int& sA22) {
    sA11 = 0; sA12 = 0; sA22 = 0;
    if (lane >= win) return;
    const int c = lane;
    const uint8_t* p = sN + WN_PITCH + c + 1;      // neighbourhood row r + 1, column c + 1 = image (iy + r, ix + c)
    int t0 = p[0], t1 = p[1];
    int dt0 = sD[c], dt1 = sD[c + 1];
    for (int r = 0; r < win; ++r) {
        const int b0 = p[(r + 1) * WN_PITCH], b1 = p[(r + 1) * WN_PITCH + 1];
        const int db0 = sD[(r + 1) * WG_PITCH + c], db1 = sD[(r + 1) * WG_PITCH + c + 1];
        const int ival = (t0 * iw00 + t1 * iw01 + b0 * iw10 + b1 * iw11 + (1 << 8)) >> 9;
        const int ixval = ((int)(short)(dt0 & 0xFFFF) * iw00 + (int)(short)(dt1 & 0xFFFF) * iw01 +
                           (int)(short)(db0 & 0xFFFF) * iw10 + (int)(short)(db1 & 0xFFFF) * iw11 + (1 << 13)) >> 14;
        const int iyval = ((dt0 >> 16) * iw00 + (dt1 >> 16) * iw01 + (db0 >> 16) * iw10 + (db1 >> 16) * iw11 + (1 << 13)) >> 14;
        sI[r * WG_PITCH + c] = (short)ival;
        sG[r * WG_PITCH + c] = (int)(((unsigned)ixval & 0xFFFFu) | ((unsigned)iyval << 16));
        sA11 += ixval * ixval;
        sA12 += ixval * iyval;
        sA22 += iyval * iyval;
        t0 = b0; t1 = b1; dt0 = db0; dt1 = db1;
    }
}

// One iteration's mismatch sums of lane c < win (zeros otherwise): J at the staged (win + 1)^2 search bytes,
// (bilinear + 2^8) >> 9, minus the template, times its derivatives, summed down column c.
KLT_HD void win_mismatch(int lane, const uint8_t* sN, const short* sI, const int* sG, int win, int iw00, int iw01, int iw10,
                         int iw11, int& sb1, int& sb2) {
    sb1 = 0; sb2 = 0;
    if (lane >= win) return;
    const int c = lane;
    const uint8_t* p = sN + c;
    int t0 = p[0], t1 = p[1];
    for (int r = 0; r < win; ++r) {
        const int b0 = p[(r + 1) * WN_PITCH], b1 = p[(r + 1) * WN_PITCH + 1];
        const int d = ((t0 * iw00 + t1 * iw01 + b0 * iw10 + b1 * iw11 + (1 << 8)) >> 9) - sI[r * WG_PITCH + c];
        const int g = sG[r * WG_PITCH + c];
        sb1 += d * (int)(short)(g & 0xFFFF);
        sb2 += d * (g >> 16);
        t0 = b0; t1 = b1;
    }
}

// ---- Host-side thresholds that let the trackers skip a division or a square root whose result is only ever compared.
//
// The minimal eigenvalue is minEig = RN(q / (2 win^2)) with q = A22 + A11 - sqrt(...), and RN(q / d) for d > 0 is
// monotone in q, so each test of minEig against a constant is a test of q against one float; likewise the forward-backward
// test sqrt(s) > fb_dist on s = dx^2 + dy^2 (double).  The thresholds are found by bisection over bit patterns with the
// host's IEEE division and square root, the same correctly rounded operations the device performs.

// the non-NaN floats in increasing order: k in [-0x7f800000, 0x7f800000] <-> -inf .. -0 (skipped), +0 .. +inf
inline float klt_key_float(long long k) {
    const uint32_t u = k >= 0 ? (uint32_t)k : 0x80000000u | (uint32_t)(-k);
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// the smallest float key in [lo, hi] where the monotone (false .. true) predicate holds; hi + 1 if it holds nowhere
template <class P> inline long long klt_first_true(long long lo, long long hi, P pred) {
    ++hi;
    while (lo < hi) {
        const long long m = lo + (hi - lo) / 2;
        if (pred(m)) hi = m; else lo = m + 1;
    }
    return lo;
}

// q < eig_q  <=>  RN(q / (2 win^2)) < min_eig, for every float q (NaN: both false)
inline float klt_eig_q(int win, float min_eig) {
    const float d = (float)(2 * win * win);
    const long long K = 0x7f800000LL;
    const long long k = klt_first_true(-K, K, [&](long long k) { return !(klt_key_float(k) / d < min_eig); });
    return klt_key_float(k);                       // the predicate holds at +inf, so k <= K
}

// q > ferr_q  <=>  RN(q / (2 win^2)) > ferr, for every float q and every ferr (NaN, infinite, negative or zero included)
inline float klt_ferr_q(int win, float ferr) {
    const float d = (float)(2 * win * win);
    const long long K = 0x7f800000LL;
    const long long k = klt_first_true(-K, K, [&](long long k) { return klt_key_float(k) / d > ferr; });
    if (k > K) return klt_key_float(K);            // never true (ferr NaN or +inf): q > +inf never holds either
    return klt_key_float(k - 1);                   // k > -K: RN(-inf / d) = -inf exceeds no ferr
}

// s > fb_s  <=>  sqrt(s) > fb_dist, for every double s >= 0 or NaN (the squared distance) and every fb_dist
inline double klt_fb_s(float fb_dist) {
    const double f = (double)fb_dist;
    const long long K = 0x7ff0000000000000LL;      // +0 .. +inf
    auto dbl = [](long long k) { double x; const uint64_t u = (uint64_t)k; memcpy(&x, &u, 8); return x; };
    const long long k = klt_first_true(0, K, [&](long long k) { return sqrt(dbl(k)) > f; });
    if (k > K) return dbl(K);                      // never true: fb_dist NaN or +inf
    if (k == 0) return -dbl(K);                    // true from 0 on (fb_dist < 0): every s >= 0 exceeds -inf
    return dbl(k - 1);
}

}  // namespace kltsetup
