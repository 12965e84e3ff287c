// F + S: grid FAST detection and sub-pixel corner refinement.
//
// Reference behaviour replaced: FeatureExtractor::detectGridFAST
// (/root/reference/src/feature_extractor.cpp:443-570).  Defined semantics = the sequential
// ascending cell order (the reference's parallel_for_ body races on `mask`, SURVEY.md 2.1).
//
//   fast_cells_kernel   (F1, one CTA per cell x frame)  FAST-9/16 score + 3x3 NMS inside each
//                       cell ROI exactly as cv::FastFeatureDetector(th, true, TYPE_9_16) on
//                       im(hroi) does (3-px dead border per cell), candidates in scan order,
//                       pre-filtered by the CV_32F-mask byte aliasing (cell-local x % 4 in {2,3}).
//                       Bound by the integer pipe: the exact score of EVERY interior pixel is
//                       computed densely, two horizontally adjacent pixels per 32-bit register
//                       (16-bit lanes) with packed (DPX) min/max.  At threshold 10 about a fifth
//                       of the pixels of a textured frame are corners, so a sparse filter +
//                       compaction in front of the score removes too little to pay for itself.
//                       On an H100 SXM (700 W limit) the three-way VIMNMX3 issues at half the rate
//                       of a two-way VIMNMX (1.7 vs 3.5 warp instructions / clock / SM), so the
//                       count that matters is two-way-equivalent min/max per pixel pair (~96).
//   fast_sweep_kernel   (F2, one CTA per frame, one warp per cell row: the wavefront of grid_sweep.cuh)  the
//                       order-dependent part: occupancy, mask discs (cv::circle midpoint rasterisation) kept as
//                       a 1-bit/pixel bitmap in shared memory, per-cell mask filter -> libstdc++ std::sort
//                       top-1 -> response >= 20 -> paint disc; adaptive nfast_th_ update (:546-552).
//   subpix_kernel       (S, one warp per point)  cv::cornerSubPix((3,3),(-1,-1),{30,0.01}).
//
// All integer work is bit-exact; S is float32/float64 with OpenCV's operation grouping
// (compiled with -fmad=false; the one FMA OpenCV uses is spelled __fmaf_rn).
#include "grid_sweep.cuh"
#include "stdsort_emul.h"
#include "tma_util.cuh"

#include <math.h>

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int MAX_CELL = 128;

// Largest number of candidates a cell of size cs can hold.  A candidate lies in the interior [3, cs - 3)^2 at cell-local
// x % 4 in {2, 3} and is a strict 3x3 maximum.  The nk = (cs - 6) / 4 + 1 column groups {4k + 2, 4k + 3} that meet the
// interior hold at most one per row (the two columns are neighbours) and none in two adjacent rows (diagonal neighbours),
// so at most ceil((cs - 6) / 2) each.  A dot lattice with one dot per group every second row reaches the bound.
__host__ __device__ constexpr int fast_cell_cap(int cs) { return ((cs - 6) / 4 + 1) * ((cs - 5) / 2); }

// FAST ring, clockwise from 12 o'clock (SURVEY.md A.1)
__host__ __device__ constexpr int ring_dx(int k) {
    constexpr int dx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    return dx[k];
}
__host__ __device__ constexpr int ring_dy(int k) { return ring_dx((k + 12) & 15); }

struct FastArgs {
    const uint8_t* img; int w, h, pitch; long long fstride;   // level 0
    int first, cs, nwc, nhc, cap;
    const int32_t* th;          // [count] threshold per frame
    uint32_t* cand;             // [count][ncells][cap]  (resp << 16) | (ky << 8) | kx
    int32_t* cand_n;            // [count][ncells]
};

// Shared-memory layout of fast_cells_kernel (bytes), shared by the kernel and its launch.
//   stage  rp x cs bytes: the staged box (TMA destination; the cell's ROI starts (x0 & 15) bytes into each row)
//   pairs  cs rows x pp words: pairs[y][x] = roi[y][x] | roi[y][x + 1] << 16, even x in words [0, hh), odd x in [hh, 2 hh)
//   sc     cs rows x scp u16: score s of a corner at th, 0 elsewhere (the 3-px border and non-corners)
//   keep   (cs - 6) rows x nk words over the stage (dead after the widening; (cs - 6)(cs - 2) < rp cs bytes): NMS survivors,
//          word k = the pixel pair x = 4k + 2, 4k + 3 (s in a survivor's lane, else 0)
struct FastSmem {
    int nk, scp, pairs, sc, bytes;
    __host__ __device__ FastSmem(int cs, int rp, int pp) {
        nk = (cs - 6) / 4 + 1;
        scp = 4 * nk + 4;                 // whole 8-byte pairs of words; word 2k + 2 of the last k stays in the row
        pairs = (rp * cs + 127) & ~127;
        sc = pairs + 4 * cs * pp;
        bytes = sc + 2 * cs * scp;
    }
};

// ---------------------------------------------------------------------------------- F1
// Per polarity: the best arc extreme over the 16 arcs of 9 contiguous ring pixels, on two pixels at once.  e[k] = d[k] + 256
// in each 16-bit lane (d = centre - ring, so every lane lies in [1, 511] and the signed s16x2 forms are exact).
// Bright (DARK = false): max over arcs of the arc minimum; dark: min over arcs of the arc maximum.  The arcs starting at 2j
// and 2j + 1 share the 8 pixels w_j = e[2j + 1 .. 2j + 8], so their better one is min(w_j, max(e[2j], e[2j + 9])) (bright):
// 8 + 8 two-way ops for the w_j (windows of 2, then 4), 8 for the end pairs, 8 three-way ops for the pair of arcs, and a
// three-way tree over the 8 pairs: 36 VIMNMX per polarity.
template <bool DARK>
__device__ __forceinline__ uint32_t best_arc(const uint32_t (&e)[16]) {
    auto in2 = [](uint32_t a, uint32_t b) { if constexpr (DARK) return __vmaxs2(a, b); else return __vmins2(a, b); };
    auto out2 = [](uint32_t a, uint32_t b) { if constexpr (DARK) return __vmins2(a, b); else return __vmaxs2(a, b); };
    auto in3 = [](uint32_t a, uint32_t b, uint32_t c) {
        if constexpr (DARK) return __vimax3_s16x2(a, b, c); else return __vimin3_s16x2(a, b, c);
    };
    auto out3 = [](uint32_t a, uint32_t b, uint32_t c) {
        if constexpr (DARK) return __vimin3_s16x2(a, b, c); else return __vimax3_s16x2(a, b, c);
    };
    uint32_t p2[8], p4[8], y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) p2[j] = in2(e[2 * j + 1], e[(2 * j + 2) & 15]);          // e[2j + 1 .. 2j + 2]
#pragma unroll
    for (int j = 0; j < 8; ++j) p4[j] = in2(p2[j], p2[(j + 1) & 7]);                    // e[2j + 1 .. 2j + 4]
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = in3(p4[j], p4[(j + 2) & 7], out2(e[2 * j], e[(2 * j + 9) & 15]));
    const uint32_t a = out3(y[0], y[1], y[2]), b = out3(y[3], y[4], y[5]);
    return out3(out3(a, b, y[6]), y[7], y[7]);
}

// HH: words per parity half of a pairs row (32 for cs <= 64, 64 above); the row pitch is a compile-time constant so every
// ring load is an immediate offset from one base register.  PP = 2 HH + 22: 22 (mod 32) makes a warp that wraps from one
// row to the next read 32 distinct banks at the default cell size 50 (22 pixel pairs per row).
// `rp`: width of the staged box (the TMA box, or the same box loaded by plain loads), a multiple of 16.
template <int HH>
__global__ void fast_cells_kernel(FastArgs A, const __grid_constant__ CUtensorMap tmap, int use_tma, int rp) {
    constexpr int PP = 2 * HH + 22;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t s_bar;
    const int cs = A.cs, tid = threadIdx.x, nthr = blockDim.x;
    const FastSmem L(cs, rp, PP);
    uint32_t* pairs = reinterpret_cast<uint32_t*>(smem + L.pairs);
    uint16_t* sc = reinterpret_cast<uint16_t*>(smem + L.sc);
    uint32_t* keep = reinterpret_cast<uint32_t*>(smem);
    const int cell = blockIdx.x, fr = blockIdx.y;
    const int r = cell / A.nwc, c = cell - r * A.nwc;
    const int x0 = c * cs, y0 = r * cs;
    int32_t* out_n = A.cand_n + (size_t)fr * (A.nwc * A.nhc) + cell;
    // cells the reference never searches (feature_extractor.cpp:510)
    if (!(x0 + cs < A.w - 1 && y0 + cs < A.h - 1)) {
        if (tid == 0) *out_n = 0;
        return;
    }
    const int th = A.th[fr];
    // a uint8 tiled box must START on a 16-byte boundary in the innermost dimension, so the box starts at x0 & ~15 and the
    // cell's ROI begins `off` bytes into each staged row.  Box columns beyond the image are zero.
    const int off = x0 & 15;
    if (use_tma && tid == 0) {
        tma::mbar_init(&s_bar, 1);
        tma::mbar_expect_tx(&s_bar, (uint32_t)(rp * cs));
        tma::load_3d(smem, &tmap, &s_bar, x0 - off, y0, A.first + fr);
    }
    {
        uint32_t* scw = reinterpret_cast<uint32_t*>(sc);
        for (int i = tid; i < cs * L.scp / 2; i += nthr) scw[i] = 0;
    }
    if (use_tma) {
        __syncthreads();             // barrier init visible to every waiter
        tma::mbar_wait_suspend(&s_bar, 0);
    } else {
        const uint8_t* img = A.img + A.fstride * (A.first + fr) + (size_t)y0 * A.pitch + (x0 - off);
        const int avail = A.w - (x0 - off);
        for (int i = tid; i < rp * cs; i += nthr) {
            const int yy = i / rp, u = i - yy * rp;
            smem[i] = u < avail ? __ldg(img + (size_t)yy * A.pitch + u) : (uint8_t)0;
        }
        __syncthreads();
    }
    // widen: pairs[y][x] for x in [0, cs); item (y, j) writes x = 2j (even half) and x = 2j + 1 (odd half) from the staged
    // bytes at u = off + 2j .. off + 2j + 2 (the odd half's entry for x = cs is never read)
    {
        const int nq = rp >> 2, hw = (cs + 1) >> 1;
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(smem);
        int y = tid / hw, j = tid - y * hw;
        const int sy = nthr / hw, sj = nthr - sy * hw;
        for (int i = tid; i < cs * hw; i += nthr) {
            const int u = off + 2 * j, q = u >> 2;
            const uint32_t* row = sw + y * nq;
            const uint32_t b4 = __funnelshift_r(row[q], row[q + 1 < nq ? q + 1 : q], 8 * (u & 3));   // bytes u .. u + 3
            uint32_t* prow = pairs + y * PP + j;
            prow[0] = __byte_perm(b4, 0u, 0x4140);
            prow[HH] = __byte_perm(b4, 0u, 0x4241);
            j += sj; y += sy;
            if (j >= hw) { j -= hw; y++; }
        }
    }
    __syncthreads();
    // score: pixel pairs (x, x + 1), x = 3 + 2j odd, over the interior [3, cs - 3)^2; an odd interior width leaves the last
    // pair half outside (its upper lane is computed from in-smem bytes and not stored)
    const int in_w = cs - 6, npair = (in_w + 1) >> 1;
    {
        const uint32_t th1 = (uint32_t)(min(max(th, -1), 255) + 257) * 0x00010001u;      // th + 257 per lane, th clamped to [-1, 255]
        int yy = tid / npair, jj = tid - yy * npair;
        const int sy = nthr / npair, sj = nthr - sy * npair;
        for (int i = tid; i < in_w * npair; i += nthr) {
            const int y = yy + 3, x = 2 * jj + 3;
            const uint32_t* ctr = pairs + y * PP + HH + (x >> 1);      // x odd: the odd half
            const uint32_t vb = ctr[0] + 0x01000100u;
            uint32_t e[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                // ring pixel (x + dx, y + dy): even dx stays in the odd half, odd dx lands in the even half
                const int dx = ring_dx(k), dy = ring_dy(k);
                const int o = dy * PP + ((dx & 1) ? -HH + ((dx + 1) >> 1) : (dx >> 1));
                e[k] = vb - ctr[o];                 // d + 256 per lane, no borrow between lanes: each lane is in [1, 511]
            }
            const uint32_t bright = best_arc<false>(e), dark = best_arc<true>(e);
            // s + 256 = max(bright, 512 - dark, 256) per lane: s = max(best bright arc, best dark arc, 0)
            const uint32_t s2 = __vimax3_s16x2(bright, 0x02000200u - dark, 0x01000100u);
            // corner at th: s > th, i.e. s + 256 >= th1 (bit 15 of each biased lane); no borrow crosses a lane
            const uint32_t ge = ((s2 | 0x80008000u) - th1) & (x + 1 < cs - 3 ? 0x80008000u : 0x00008000u);
            const uint32_t sv = (s2 - 0x01000100u) & ((ge >> 15) * 0xFFFFu);
            uint16_t* o = sc + y * L.scp + x;
            o[0] = (uint16_t)sv;
            o[1] = (uint16_t)(sv >> 16);                           // 0 for the upper half of a half pair (outside the interior)
            jj += sj; yy += sy;
            if (jj >= npair) { jj -= npair; yy++; }
        }
    }
    __syncthreads();
    // 3x3 NMS on response = s - 1 (non-corners count 0), strictly greater than all 8 neighbours: s > max(neighbours' s, 1).
    // Only cell-local x % 4 in {2, 3} (the CV_32F mask read as bytes): one keep word per pixel pair x = 4k + 2, 4k + 3,
    // which is sc word 2k + 1 of its row.
    const int nk = L.nk, nkeep = in_w * nk, scw = L.scp / 2;
    {
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(sc);
        int yy = tid / nk, kk = tid - yy * nk;
        const int sy = nthr / nk, sk = nthr - sy * nk;
        for (int t = tid; t < nkeep; t += nthr) {
            const uint32_t* w = s32 + (yy + 3) * scw + 2 * kk;
            const uint2 a0 = *reinterpret_cast<const uint2*>(w - scw), a1 = *reinterpret_cast<const uint2*>(w),
                        a2 = *reinterpret_cast<const uint2*>(w + scw);
            const uint32_t ca = __vimax3_u16x2(a0.x, a1.x, a2.x);                 // column maxima at x = 4k, 4k + 1
            const uint32_t cc = __vimax3_u16x2(w[2 - scw], w[2], w[2 + scw]);    // at x = 4k + 4, 4k + 5
            const uint32_t vb = __vmaxu2(a0.y, a2.y);                            // above / below x = 4k + 2, 4k + 3
            const uint32_t cb = __vmaxu2(vb, a1.y);
            const uint32_t left = __byte_perm(ca, cb, 0x5432), right = __byte_perm(cb, cc, 0x5432);   // x - 1, x + 1
            const uint32_t m = __vimax3_u16x2(__vimax3_u16x2(left, right, vb), 0x00010001u, 0x00010001u);
            const uint32_t s = a1.y;
            const uint32_t gt = ((s | 0x80008000u) - (m + 0x00010001u)) & 0x80008000u;   // bit 15 of a lane: s > m
            keep[t] = s & ((gt >> 15) * 0xFFFFu);
            kk += sk; yy += sy;
            if (kk >= nk) { kk -= nk; yy++; }
        }
    }
    __syncthreads();
    // ordered emission (row-major scan order) by warp 0, 32 keep words per step
    if (tid < 32) {
        uint32_t* out = A.cand + ((size_t)fr * (A.nwc * A.nhc) + cell) * A.cap;
        const int lane = tid;
        const unsigned below = (1u << lane) - 1u;
        const unsigned rnk = 0xFFFFFFFFu / (unsigned)nk + 1u;          // ceil(2^32 / nk): t / nk == umulhi(t, rnk) for t < 2^16, nk > 1
        int n = 0;
        for (int base = 0; base < nkeep; base += 32) {
            const uint32_t w = base + lane < nkeep ? keep[base + lane] : 0u;
            const uint32_t s0 = w & 0xFFFFu, s1 = w >> 16;
            const unsigned m0 = __ballot_sync(FULL, s0 != 0u), m1 = __ballot_sync(FULL, s1 != 0u);
            if (w) {
                const int p = n + __popc(m0 & below) + __popc(m1 & below);
                const unsigned t = base + lane, yy = nk > 1 ? __umulhi(t, rnk) : t, kk = t - yy * nk;
                const uint32_t yx = ((yy + 3u) << 8) | (4u * kk + 2u);
                // n never exceeds fast_cell_cap(cs), so every candidate has a slot
                if (s0) out[p] = ((s0 - 1u) << 16) | yx;
                if (s1) out[p + (s0 != 0u)] = ((s1 - 1u) << 16) | (yx + 1u);
            }
            n += __popc(m0) + __popc(m1);
        }
        if (lane == 0) *out_n = n;
    }
}

// ---------------------------------------------------------------------------------- F2
// Sort keys are (response << 16) | candidate index (stdsort_emul.h).
constexpr int SKEY_SHIFT = 16;
constexpr int SKEY_IDX = (1 << SKEY_SHIFT) - 1;
// fast_sweep_kernel holds up to WAVE_REG_CAND candidates of a cell in registers (four per lane) and their sort keys in
// shared memory; a cell with more candidates reads them from the list and sorts in a global area (SweepArgs::skey_g).
constexpr int WAVE_REG_CAND = 128;

struct SweepArgs : gsweep::SweepBase {
    int cap, max_per_frame;
    int* skey_g;                     // [count][warps][cap] sort keys of cells with > WAVE_REG_CAND candidates
    const uint32_t* cand; const int32_t* cand_n;
    int32_t* th;                     // in/out per frame
    int2* out_int;                   // [count][max_per_frame]
    int32_t* out_n;                  // [count]
};

// Shared-memory layout of fast_sweep_kernel: min(cap, WAVE_REG_CAND) sort keys per warp between the bitmap and the counters.
constexpr int FSWEEP_MAX_WARPS = 16;
__host__ __device__ inline gsweep::SweepSmem fast_sweep_smem(int w, int h, int nwc, int nhc, int cap, int nwarps) {
    return gsweep::SweepSmem(w, h, nwc, nhc, nwarps, nwarps * min(cap, WAVE_REG_CAND) * 4, alignof(int));
}

// The wavefront sweep of grid_sweep.cuh, one warp per cell row: exactly the sequential result in nwc + 2 nhc cell times
// instead of nwc * nhc (pure latency; 0.070 ms, 3.5 % of the C2 step, on an H100 SXM at 700 W).  As many warps as the
// shared memory allows, up to one per cell row (at most FSWEEP_MAX_WARPS).  Cell c's detection goes to slot c of the
// frame's output (max_per_frame >= ncells), and the slots are compacted in cell order at the end.
__global__ void __launch_bounds__(FSWEEP_MAX_WARPS * 32, 1) fast_sweep_kernel(SweepArgs A) {
    extern __shared__ __align__(16) uint8_t sm[];
    const int tid = threadIdx.x, fr = blockIdx.x, nthreads = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nthreads >> 5;
    const int ncells = A.nwc * A.nhc;
    const gsweep::SweepSmem L = fast_sweep_smem(A.w, A.h, A.nwc, A.nhc, A.cap, nwarps);
    const int wpr = L.wpr;
    uint32_t* bm = reinterpret_cast<uint32_t*>(sm);
    const int nskey = min(A.cap, WAVE_REG_CAND);
    int* skey_sm = reinterpret_cast<int*>(sm + L.mid) + warp * nskey;
    volatile int* progress = gsweep::progress_counters(L, sm);
    const uint8_t* occ = sm + L.occ;
    int* skey_big = A.skey_g ? A.skey_g + ((size_t)fr * nwarps + warp) * A.cap : nullptr;
    gsweep::init_mask(A, L, sm, fr);
    const uint32_t* cand = A.cand + (size_t)fr * ncells * A.cap;
    const int32_t* cand_n = A.cand_n + (size_t)fr * ncells;
    int2* out = A.out_int + (size_t)fr * A.max_per_frame;
    // A cell's candidates do not depend on any other cell, and the row's cell-to-cell chain is what the frame waits for: the
    // count and the first WAVE_REG_CAND candidates of cell c + 2 are requested (five independent loads; the list's slots past
    // the count are allocated, and dropped below) before cell c is worked on, so no global-memory latency is left in the chain.
    struct CellFetch { int n; uint32_t v[4]; };
    auto fetch = [&](int r, int c) {
        CellFetch f = {0, {0u, 0u, 0u, 0u}};
        if (c < A.nwc) {
            const int cell = r * A.nwc + c;
            f.n = __ldg(cand_n + cell);
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (32 * q + lane < A.cap) f.v[q] = __ldg(cand + (size_t)cell * A.cap + 32 * q + lane);
        }
        return f;
    };
    for (int r = warp; r < A.nhc; r += nwarps) {
        CellFetch f0 = fetch(r, 0), f1 = fetch(r, 1);
        for (int c = 0; c < A.nwc; ++c) {
            const CellFetch cur = f0;
            f0 = f1;
            f1 = fetch(r, c + 2);
            const int cell = r * A.nwc + c;
            const int x0 = c * A.cs, y0 = r * A.cs;
            const bool search = !occ[r * (A.nwc + 1) + c] && (x0 + A.cs < A.w - 1 && y0 + A.cs < A.h - 1);
            const int n = search ? cur.n : 0;
            const uint32_t* ccand = cand + (size_t)cell * A.cap;
            uint32_t cdv[4];                                                   // the first WAVE_REG_CAND: four per lane
#pragma unroll
            for (int q = 0; q < 4; ++q) cdv[q] = 32 * q + lane < n ? cur.v[q] : 0u;
            gsweep::wave_wait(progress, nwarps, r, c, A.nwc);
            int2 det = make_int2(-1, -1);
            if (n > 0) {
                // mask filter + ordered compaction of survivors into skey (shared memory, or the global area for big cells)
                const bool big = n > WAVE_REG_CAND;                            // uniform
                int* skey = big ? skey_big : skey_sm;
                int ns = 0, vmax = -1;
                auto filter = [&](uint32_t cd, int j) {
                    bool ok = false;
                    if (j < n) {
                        const int kx = cd & 255, ky = (cd >> 8) & 255;
                        const int mx = x0 + (kx >> 2), my = y0 + ky;
                        ok = ((bm[(size_t)my * wpr + (mx >> 5)] >> (mx & 31)) & 1u) == 0;
                    }
                    const unsigned m = __ballot_sync(FULL, ok);
                    if (ok) {
                        const int pos = ns + __popc(m & ((1u << lane) - 1));
                        skey[pos] = (int)((cd >> 16) << SKEY_SHIFT) | j;       // (response << 16) | candidate index
                        vmax = max(vmax, (int)(cd >> 16));
                    }
                    ns += __popc(m);
                };
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (32 * q >= n) break;                                    // uniform
                    filter(cdv[q], 32 * q + lane);
                }
                for (int base = WAVE_REG_CAND; base < n; base += 32) {         // big cells only
                    const int j = base + lane;
                    filter(j < n ? __ldg(ccand + j) : 0u, j);
                }
                if (ns > 0) {
                    vmax = __reduce_max_sync(FULL, vmax);
                    __syncwarp();
                    int nmax = 0, firstmax = 0x7fffffff;
                    for (int base = 0; base < ns; base += 32) {
                        const int j = base + lane;
                        const bool is = j < ns && (skey[j] >> SKEY_SHIFT) == vmax;
                        const unsigned m = __ballot_sync(FULL, is);
                        if (m && firstmax == 0x7fffffff) firstmax = base + __ffs(m) - 1;
                        nmax += __popc(m);
                    }
                    int win_j;
                    if (nmax == 1 || ns <= 16) {
                        win_j = skey[firstmax] & SKEY_IDX;                     // unique maximum / libstdc++'s insertion-sort range
                    } else {
                        if (lane == 0) ov2sort::sort_desc_front(skey, ns);     // only skey[0] is read
                        __syncwarp();
                        win_j = skey[0] & SKEY_IDX;
                    }
                    __syncwarp();
                    if (vmax >= 20) {                                          // vkps.at(0).response >= 20
                        const int wq = win_j >> 5;                              // uniform
                        const uint32_t mine = wq == 0 ? cdv[0] : (wq == 1 ? cdv[1] : (wq == 2 ? cdv[2] : cdv[3]));
                        const uint32_t cd = win_j < WAVE_REG_CAND ? __shfl_sync(FULL, mine, win_j & 31) : __ldg(ccand + win_j);
                        det = make_int2(x0 + (int)(cd & 255), y0 + (int)((cd >> 8) & 255));
                        gsweep::paint_disc(A, bm, wpr, det.x, det.y, lane, 32);
                        __syncwarp();
                    }
                }
            }
            if (lane == 0) out[cell] = det;
            gsweep::wave_publish(progress, nwarps, r, c, lane);
        }
    }
    __syncthreads();
    // compaction in cell order + the adaptive threshold (feature_extractor.cpp:546-552).  A detection only moves left, so
    // each round reads its 128 slots (four loads in flight, one L2 latency) before it writes any of them.
    if (warp == 0) {
        int nbkps = 0, nbempty = 0;
        for (int base = 0; base < ncells; base += 128) {
            int2 d[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int cell = base + 32 * q + lane;
                d[q] = cell < ncells ? out[cell] : make_int2(-1, -1);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int cell = base + 32 * q + lane;
                const int r = cell / A.nwc, c = cell - r * A.nwc;
                const bool empty = cell < ncells && !occ[r * (A.nwc + 1) + c], has = d[q].x >= 0;
                const unsigned mh = __ballot_sync(FULL, has);
                if (has) out[nbkps + __popc(mh & ((1u << lane) - 1))] = d[q];
                nbkps += __popc(mh);
                nbempty += __popc(__ballot_sync(FULL, empty));
            }
        }
        for (int i = nbkps + lane; i < A.max_per_frame; i += 32) out[i] = make_int2(-1, -1);
        if (lane == 0) {
            A.out_n[fr] = nbkps;
            int th = A.th[fr];
            if ((double)nbkps < 0.5 * (double)nbempty && nbempty > 10) th = (int)((double)th * 0.66);
            else if (nbkps == nbempty) th = (int)((double)th * 1.5);
            A.th[fr] = th;
        }
    }
}

// ---------------------------------------------------------------------------------- S
struct SubpixArgs {
    const uint8_t* img; int w, h, pitch; long long fstride;
    int first, max_per_frame, n;   // n = count * max_per_frame
    const int2* in_int;
    float2* out;
    int do_subpix;
    float mask[49];                // exp(-(i/3)^2) * exp(-(j/3)^2), computed on the host with libm expf
    int32_t* iters;                // COUNT instantiation only: iterations run per slot (-1: empty slot)
};

// cv::getRectSubPix(8u -> 32f, 9x9) value at patch (i, j); grouping found by probing cv2 4.13
// (oracle/image_ref.py::_get_rect_subpix_9).
__device__ __forceinline__ float rect_subpix_px(const uint8_t* img, int pitch, int W, int H, int ix, int iy, float a,
                                                float b, int i, int j) {
    const bool inside = 0 <= ix && ix + 9 < W && 0 <= iy && iy + 9 < H;
    const float a11 = (1.f - a) * (1.f - b), a12 = a * (1.f - b), a21 = (1.f - a) * b, a22 = a * b;
    if (inside) {
        const uint8_t* p = img + (size_t)(iy + i) * pitch + ix + j;
        float p00 = p[0], p01 = p[1], p10 = p[pitch], p11 = p[pitch + 1];
        return (p00 * a11 + p01 * a12) + (p10 * a21 + p11 * a22);
    }
    const int rx = ix < 0 ? min(-ix, 9) : 0;
    const int rw = ix < W - 9 ? 9 : max(W - ix - 1, 0);
    const int ry = iy < 0 ? -iy : 0;
    const int rh = iy < H - 9 ? 9 : max(H - iy - 1, 0);
    const int r0 = clampi(iy + i, 0, H - 1), r1 = clampi(iy + i + 1, 0, H - 1);
    const uint8_t* s0 = img + (size_t)r0 * pitch;
    const uint8_t* s1 = img + (size_t)r1 * pitch;
    if (j < rx || j >= rw) {
        int cc = j < rx ? 0 : (i < ry ? W - 2 : W - 1);
        cc = clampi(cc, 0, W - 1);
        return (float)s0[cc] * (1.f - b) + (float)s1[cc] * b;
    }
    const int cc = ix + j;
    if (i < ry || i >= rh) return __fmaf_rn((float)s0[cc + 1], a, (float)s0[cc] * (1.f - a));
    return ((float)s0[cc] * a11 + (float)s0[cc + 1] * a12) + ((float)s1[cc] * a21 + (float)s1[cc + 1] * a22);
}

// One warp per point.  The 9 x 9 getRectSubPix patch only needs the 10 x 10 pixels at the centre's integer origin (ix, iy),
// and successive iterations move the centre by a fraction of a pixel: the pixels are staged in shared memory (as floats)
// when the origin changes and re-interpolated from there otherwise.  Every lane keeps fixed patch and gradient
// positions, so no division is left in the loop.  Expressions and summation order are those of cv::cornerSubPix.
template <bool COUNT>
__global__ void __launch_bounds__(128) subpix_kernel(SubpixArgs A) {
    __shared__ float sraw[4][100];
    __shared__ float spatch[4][81];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int idx = blockIdx.x * 4 + warp;
    if (idx >= A.n) return;
    const int2 ip = A.in_int[idx];
    if (ip.x < 0) {
        if (lane == 0) A.out[idx] = make_float2(-1.f, -1.f);
        if (COUNT && lane == 0) A.iters[idx] = -1;
        return;
    }
    const float2 cT = make_float2((float)ip.x, (float)ip.y);
    if (!A.do_subpix) {
        if (lane == 0) A.out[idx] = cT;
        if (COUNT && lane == 0) A.iters[idx] = 0;
        return;
    }
    const int fr = idx / A.max_per_frame;
    const uint8_t* img = A.img + A.fstride * (A.first + fr);
    float* sp = spatch[warp];
    float* raw = sraw[warp];
    // patch pixels lane, lane + 32, lane + 64 (the last for lanes 0..16): position in the 10-wide staged block
    const int r0 = lane + lane / 9, r1 = lane + 32 + (lane + 32) / 9, r2 = lane + 64 + (lane + 64) / 9;   // p + p / 9
    const bool has2 = lane + 64 < 81;
    // gradient pixels lane and lane + 32 (the second for lanes 0..16)
    const int gi0 = lane / 7, gj0 = lane % 7;
    const int gi1 = (lane + 32) / 7, gj1 = (lane + 32) % 7;
    const bool hasg1 = lane + 32 < 49;
    const float* q0 = sp + (gi0 + 1) * 9 + (gj0 + 1);
    const float* q1 = sp + (hasg1 ? (gi1 + 1) * 9 + (gj1 + 1) : 10);
    const float mf0 = A.mask[lane], mf1 = hasg1 ? A.mask[lane + 32] : 0.f;
    const float pxf0 = (float)(gj0 - 3), pyf0 = (float)(gi0 - 3), pxf1 = (float)(gj1 - 3), pyf1 = (float)(gi1 - 3);
    float2 cI = cT;
    const double eps = 0.01 * 0.01;
    int iter = 0, nrun = 0;
    int sx = -1, sy = -1;                                       // origin of the staged block (never negative)
    double err = 0.0;
    do {
        ++nrun;
        const float x = cI.x - 4.f, y = cI.y - 4.f;
        const int ix = __float2int_rd(x), iy = __float2int_rd(y);
        const float a = x - (float)ix, b = y - (float)iy;
        __syncwarp();
        if (0 <= ix && ix + 9 < A.w && 0 <= iy && iy + 9 < A.h) {
            if (ix != sx || iy != sy) {
                const uint8_t* p = img + (size_t)iy * A.pitch + ix;
                for (int e = lane; e < 100; e += 32) {
                    const int rr = e / 10;
                    raw[e] = (float)p[(size_t)rr * A.pitch + (e - rr * 10)];
                }
                sx = ix; sy = iy;
                __syncwarp();
            }
            const float a11 = (1.f - a) * (1.f - b), a12 = a * (1.f - b), a21 = (1.f - a) * b, a22 = a * b;
            sp[lane] = (raw[r0] * a11 + raw[r0 + 1] * a12) + (raw[r0 + 10] * a21 + raw[r0 + 11] * a22);
            sp[lane + 32] = (raw[r1] * a11 + raw[r1 + 1] * a12) + (raw[r1 + 10] * a21 + raw[r1 + 11] * a22);
            if (has2) sp[lane + 64] = (raw[r2] * a11 + raw[r2 + 1] * a12) + (raw[r2 + 10] * a21 + raw[r2 + 11] * a22);
        } else {
            // within 4 px of a border: getRectSubPix's border rules, pixel by pixel
            for (int p = lane; p < 81; p += 32) sp[p] = rect_subpix_px(img, A.pitch, A.w, A.h, ix, iy, a, b, p / 9, p % 9);
        }
        __syncwarp();
        double sa = 0, sb = 0, scc = 0, sbb1 = 0, sbb2 = 0;
        {
            const double m0 = (double)mf0, px0 = (double)pxf0, py0 = (double)pyf0;
            const double tgx = (double)(q0[1] - q0[-1]);
            const double tgy = (double)(q0[9] - q0[-9]);
            const double gxx = tgx * tgx * m0, gxy = tgx * tgy * m0, gyy = tgy * tgy * m0;
            sa += gxx; sb += gxy; scc += gyy;
            sbb1 += gxx * px0 + gxy * py0;
            sbb2 += gxy * px0 + gyy * py0;
        }
        if (hasg1) {
            const double m1 = (double)mf1, px1 = (double)pxf1, py1 = (double)pyf1;
            const double tgx = (double)(q1[1] - q1[-1]);
            const double tgy = (double)(q1[9] - q1[-9]);
            const double gxx = tgx * tgx * m1, gxy = tgx * tgy * m1, gyy = tgy * tgy * m1;
            sa += gxx; sb += gxy; scc += gyy;
            sbb1 += gxx * px1 + gxy * py1;
            sbb2 += gxy * px1 + gyy * py1;
        }
        // The five warp sums, each the xor butterfly's tree ((x[i] + x[i ^ 16]) + ...: order 16, 8, 4, 2, 1), with the sums
        // spread over the lanes instead of repeated in all of them: at 16 the lower half-warp goes on with sa and scc, the
        // upper with sb and sbb1; at 8 lanes with bit 3 clear keep the first of their two, the others the second; at 4 lanes
        // with bit 2 set take over sbb2.  A lane adds the same two partial sums the butterfly adds there (a + b = b + a), so
        // every sum has the butterfly's bits with 8 shuffles in place of 25; lanes 0, 16, 8, 24 and 4 hold the results.
        const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
        double u = (h16 ? sb : sa) + __shfl_xor_sync(FULL, h16 ? sa : sb, 16);        // sa | sb
        double v = (h16 ? sbb1 : scc) + __shfl_xor_sync(FULL, h16 ? scc : sbb1, 16);  // scc | sbb1
        sbb2 += __shfl_xor_sync(FULL, sbb2, 16);
        u = (h8 ? v : u) + __shfl_xor_sync(FULL, h8 ? u : v, 8);                      // sa | sb | scc | sbb1 by bits 4, 3
        sbb2 += __shfl_xor_sync(FULL, sbb2, 8);
        u = (h4 ? sbb2 : u) + __shfl_xor_sync(FULL, h4 ? u : sbb2, 4);
        u += __shfl_xor_sync(FULL, u, 2);
        u += __shfl_xor_sync(FULL, u, 1);
        sa = __shfl_sync(FULL, u, 0); sb = __shfl_sync(FULL, u, 16); scc = __shfl_sync(FULL, u, 8);
        sbb1 = __shfl_sync(FULL, u, 24); sbb2 = __shfl_sync(FULL, u, 4);
        const double det = sa * scc - sb * sb;
        if (fabs(det) <= 2.220446049250313e-16 * 2.220446049250313e-16) break;
        const double scale = 1.0 / det;
        float2 cI2;
        cI2.x = (float)((double)cI.x + scc * scale * sbb1 - sb * scale * sbb2);
        cI2.y = (float)((double)cI.y - sb * scale * sbb1 + sa * scale * sbb2);
        const float ex = cI2.x - cI.x, ey = cI2.y - cI.y;
        err = (double)(ex * ex + ey * ey);
        if (cI2.x < 0 || cI2.x >= (float)A.w || cI2.y < 0 || cI2.y >= (float)A.h) break;
        cI = cI2;
    } while (++iter < 30 && err > eps);
    if (fabsf(cI.x - cT.x) > 3.f || fabsf(cI.y - cT.y) > 3.f) cI = cT;
    if (lane == 0) A.out[idx] = cI;
    if (COUNT && lane == 0) A.iters[idx] = nrun;
}

// cornerSubPix's 7 x 7 weights, exactly as OpenCV forms them
void subpix_mask(float* mask) {
    for (int i = 0; i < 7; ++i) {
        float y = (float)(i - 3) / 3;
        float vy = expf(-y * y);
        for (int j = 0; j < 7; ++j) {
            float x = (float)(j - 3) / 3;
            mask[i * 7 + j] = (float)(vy * expf(-x * x));
        }
    }
}

}  // namespace

template <int HH>
static ov2_status launch_fast_cells_hh(ov2_ctx* ctx, const FastArgs& FA, int nframes_grid, const CUtensorMap& tmap, int use_tma,
                                      int rp) {
    const int cs = FA.cs;
    const int threads = cs > 24 ? 128 : 32;
    const FastSmem L(cs, rp, 2 * HH + 22);
    if (L.bytes > 48 * 1024)
        OV2_CUDA(ctx, cudaFuncSetAttribute(fast_cells_kernel<HH>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.bytes));
    OV2_LAUNCH(ctx, "fast_cells_kernel",
               fast_cells_kernel<HH><<<dim3(FA.nwc * FA.nhc, nframes_grid), threads, L.bytes, ctx->stream>>>(FA, tmap, use_tma, rp));
    return OV2_OK;
}

// TMA staging: a 3-D tiled tensor map {W, H, frames} over the level-0 images, box {rp, cs, 1} (rp = cs + 15 rounded up to
// 16 bytes: the box starts on the 16-byte boundary at or below the cell).  Plain loads of the same box when the images do
// not meet the TMA alignment rules (user-aliased level 0 with an odd pitch or base) or the driver lacks the encoder.
static ov2_status launch_fast_cells(ov2_ctx* ctx, const ov2_pyr* pyr, const FastArgs& FA, int nframes_grid) {
    const int cs = FA.cs;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    const int rp = (cs + 15 + 15) & ~15;      // staged box width, TMA or not
    const int use_tma = tma::make_u8_3d(&tmap, FA.img, FA.w, FA.h, pyr->batch, FA.pitch, FA.fstride, rp, cs) ? 1 : 0;
    return cs <= 64 ? launch_fast_cells_hh<32>(ctx, FA, nframes_grid, tmap, use_tma, rp)
                    : launch_fast_cells_hh<64>(ctx, FA, nframes_grid, tmap, use_tma, rp);
}


extern "C" ov2_status ov2_grid_fast(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int cellsize,
                                    const int32_t* curkp_offsets, const float* curkps, int32_t* fast_th_inout,
                                    int max_per_frame, float* out_pts, int32_t* out_counts, int32_t* out_pts_int,
                                    int do_subpix) {
    if (!ctx || !pyr || !pyr->l0 || first < 0 || count <= 0 || first + count > pyr->batch || !fast_th_inout ||
        !out_pts || !out_counts)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_grid_fast: bad arguments");
    if (cellsize < 8 || cellsize > MAX_CELL)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_grid_fast: cellsize must be in [8, 128]");
    const int W = pyr->w[0], H = pyr->h[0];
    const int nwc = W / cellsize, nhc = H / cellsize, ncells = nwc * nhc;
    if (ncells == 0 || max_per_frame < ncells)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_grid_fast: max_per_frame < number of cells");
    const int cap = fast_cell_cap(cellsize);
    // sweep warps: one per cell row, up to FSWEEP_MAX_WARPS, as many as fit the shared memory
    int nw = nhc < FSWEEP_MAX_WARPS ? nhc : FSWEEP_MAX_WARPS;
    while (nw > 1 && fast_sweep_smem(W, H, nwc, nhc, cap, nw).bytes > gsweep::SMEM_LIMIT) --nw;
    const size_t smem = fast_sweep_smem(W, H, nwc, nhc, cap, nw).bytes;
    if (smem > gsweep::SMEM_LIMIT)
        return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_grid_fast: image too large for the shared-memory mask bitmap");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    DetectArgs<int32_t> D;
    if ((st = stage_detect_args(ctx, "ov2_grid_fast", count, max_per_frame, curkp_offsets, curkps, fast_th_inout, out_pts,
                                out_counts, out_pts_int, &D)) != OV2_OK)
        return st;
    uint32_t* d_cand = nullptr;
    int32_t* d_candn = nullptr;
    if ((st = ov2_scratch(ctx, (size_t)count * ncells * cap, d_cand)) != OV2_OK) return st;
    if ((st = ov2_scratch(ctx, (size_t)count * ncells, d_candn)) != OV2_OK) return st;
    int* d_skey = nullptr;      // sort keys of the cells with more candidates than the sweep keeps in registers
    if (cap > WAVE_REG_CAND && (st = ov2_scratch(ctx, (size_t)count * nw * cap, d_skey)) != OV2_OK) return st;

    FastArgs FA;
    FA.img = pyr->l0; FA.w = W; FA.h = H; FA.pitch = (int)pyr->l0_pitch; FA.fstride = (long long)pyr->l0_fstride;
    FA.first = first; FA.cs = cellsize; FA.nwc = nwc; FA.nhc = nhc; FA.cap = cap;
    FA.th = D.state; FA.cand = d_cand; FA.cand_n = d_candn;
    if ((st = launch_fast_cells(ctx, pyr, FA, count)) != OV2_OK) return st;
    SweepArgs SA;
    gsweep::init_base(SA, W, H, cellsize, D.kp_off, D.kps);
    SA.cap = cap; SA.max_per_frame = max_per_frame; SA.skey_g = d_skey;
    SA.cand = d_cand; SA.cand_n = d_candn; SA.th = D.state; SA.out_int = D.ints; SA.out_n = D.cnt;
    static size_t smem_attr[16] = {0};
    if (smem > 48 * 1024 && smem > smem_attr[ctx->device & 15]) {
        OV2_CUDA(ctx, cudaFuncSetAttribute(fast_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_attr[ctx->device & 15] = smem;
    }
    OV2_LAUNCH(ctx, "fast_sweep_kernel", fast_sweep_kernel<<<count, nw * 32, smem, ctx->stream>>>(SA));
    if ((st = ov2_subpix_launch(ctx, pyr, first, count, max_per_frame, D.ints, D.out, do_subpix, nullptr)) != OV2_OK) return st;
    return ov2_end(ctx);
}

extern "C" int ov2_fast_cell_capacity(int cellsize) {
    return cellsize < 8 || cellsize > MAX_CELL ? 0 : fast_cell_cap(cellsize);
}

// Test hook: the per-cell FAST candidate lists of one frame (stage F1 only), so the tests can
// pin cv::FastFeatureDetector parity cell by cell.  cand_out: ncells*cap words
// ((response << 16) | (y << 8) | x, cell-local), cand_n_out: ncells counts; *cap_out = capacity used.
extern "C" ov2_status ov2_debug_fast_cells(ov2_ctx* ctx, const ov2_pyr* pyr, int frame, int cellsize, int fast_th,
                                           uint32_t* cand_out, int32_t* cand_n_out, int cap_in, int* cap_out) {
    if (!ctx || !pyr || !pyr->l0 || frame < 0 || frame >= pyr->batch || cellsize < 8 || cellsize > MAX_CELL)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_debug_fast_cells: bad arguments");
    const int W = pyr->w[0], H = pyr->h[0];
    const int nwc = W / cellsize, nhc = H / cellsize, ncells = nwc * nhc;
    const int cap = fast_cell_cap(cellsize);
    if (cap_out) *cap_out = cap;
    if (cap_in < cap) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_debug_fast_cells: cap_in too small");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    FastArgs FA;
    FA.img = pyr->l0; FA.w = W; FA.h = H; FA.pitch = (int)pyr->l0_pitch; FA.fstride = (long long)pyr->l0_fstride;
    FA.first = frame; FA.cs = cellsize; FA.nwc = nwc; FA.nhc = nhc; FA.cap = cap;
    int32_t* d_th = nullptr;
    if ((st = ov2_scratch(ctx, 1, d_th)) != OV2_OK) return st;
    OV2_CUDA(ctx, cudaMemcpyAsync(d_th, &fast_th, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    FA.th = d_th;
    if ((st = ov2_stage_out(ctx, cand_out, (size_t)ncells * cap, FA.cand)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, cand_n_out, (size_t)ncells, FA.cand_n)) != OV2_OK) return st;
    if ((st = launch_fast_cells(ctx, pyr, FA, 1)) != OV2_OK) return st;
    return ov2_end(ctx);
}

ov2_status ov2_subpix_launch(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int max_per_frame, const int2* d_int,
                             float2* d_out, int do_subpix, int32_t* d_iters) {
    SubpixArgs PA;
    PA.img = pyr->l0; PA.w = pyr->w[0]; PA.h = pyr->h[0]; PA.pitch = (int)pyr->l0_pitch; PA.fstride = (long long)pyr->l0_fstride;
    PA.first = first; PA.max_per_frame = max_per_frame; PA.n = count * max_per_frame;
    PA.in_int = d_int; PA.out = d_out; PA.do_subpix = do_subpix;
    PA.iters = d_iters;
    subpix_mask(PA.mask);
    if (d_iters)
        OV2_LAUNCH(ctx, "subpix_kernel", subpix_kernel<true><<<div_up(PA.n, 4), 128, 0, ctx->stream>>>(PA));
    else
        OV2_LAUNCH(ctx, "subpix_kernel", subpix_kernel<false><<<div_up(PA.n, 4), 128, 0, ctx->stream>>>(PA));
    return OV2_OK;
}

// Measurement hook: cornerSubPix on `pts_int` (count * max_per_frame slots, x < 0: empty) as ov2_grid_fast runs it,
// returning the number of iterations each point took.  A second instantiation of the kernel: the product launch
// carries no counter.
extern "C" ov2_status ov2_debug_subpix_iters(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int max_per_frame,
                                             const int32_t* pts_int, float* out_pts, int32_t* iters_out) {
    if (!ctx || !pyr || !pyr->l0 || first < 0 || count <= 0 || first + count > pyr->batch || max_per_frame <= 0 || !pts_int ||
        !out_pts || !iters_out)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_debug_subpix_iters: bad arguments");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    const size_t n = (size_t)count * max_per_frame;
    const int2* d_int = nullptr;
    float2* d_out = nullptr;
    int32_t* d_iters = nullptr;
    if ((st = ov2_stage_in(ctx, pts_int, n, d_int)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, out_pts, n, d_out)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, iters_out, n, d_iters)) != OV2_OK) return st;
    if ((st = ov2_subpix_launch(ctx, pyr, first, count, max_per_frame, d_int, d_out, 1, d_iters)) != OV2_OK) return st;
    return ov2_end(ctx);
}
