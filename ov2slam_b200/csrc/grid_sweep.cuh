// The sweep machinery both grid detectors share (grid FAST, frontend_fast.cu; detectSingleScale, frontend_sscale.cu).
//
// The reference walks the cells in row-major order and every detection paints a disc of radius cs / 4 into the mask, so a
// cell depends on the cells before it - but a disc reaches at most cs / 4 pixels into the NEIGHBOURING cells.  Cell (r, c)
// therefore only needs (r, c-1), (r-1, c-1), (r-1, c) and (r-1, c+1) to be finished: one WARP per cell row, row r trailing
// row r-1 by two cells (wavefront), gives exactly the sequential result in (nwc + 2 nhc) cell times instead of nwc * nhc.
// progress[r] = number of cells of row r that are finished (volatile shared memory; discs are painted with shared atomics
// before the counter moves).  With one warp the rows run in order and there are no counters.
#pragma once

#include "ov2_common.cuh"

namespace gsweep {

constexpr int MAX_RADIUS = 32;                   // cs / 4 for cells up to 128
constexpr size_t SMEM_LIMIT = 227 * 1024;        // opt-in dynamic shared memory of one block (sm_90)

// The fields of a sweep's kernel arguments that the shared pieces read.
struct SweepBase {
    int w, h, cs, nwc, nhc, radius;
    int hw[MAX_RADIUS + 1];          // cv::circle half-widths per |dy|
    const int32_t* kp_off;           // [count+1] or NULL
    const float2* kps;               // existing keypoints
};

// Shared-memory layout of a sweep (byte offsets): the mask bitmap (h rows of wpr words, bit = 1: mask is 0.0f there), `mid`
// bytes of the sweep's own data (aligned to mid_align, a power of two >= 4), row progress counters (nhc ints, only when more than one warp sweeps) and
// the occupancy grid ((nhc+1) x (nwc+1) bytes).  The host sizes in size_t, so that no image size can wrap its refusal; a
// kernel only runs a layout the host accepted (bytes <= SMEM_LIMIT) and computes it in int, which keeps the sweeps' 64-bit
// registers for their loops.
struct SweepSmem {
#ifdef __CUDA_ARCH__
    using off = int;
#else
    using off = size_t;
#endif
    int wpr;
    off mid, progress, occ, bytes;
    __host__ __device__ SweepSmem(int w, int h, int nwc, int nhc, int nwarps, off mid_bytes, int mid_align) {
        wpr = (w + 31) >> 5;
        mid = ((off)h * wpr * 4 + mid_align - 1) & ~(off)(mid_align - 1);
        progress = mid + mid_bytes;
        occ = progress + (nwarps > 1 ? (off)nhc * 4 : 0);
        bytes = (occ + (off)(nhc + 1) * (nwc + 1) + 15) & ~(off)15;
    }
};

// OpenCV's filled-circle rasterisation (midpoint algorithm): half-width per |dy|
inline void circle_halfwidths(int radius, int* hw) {
    for (int i = 0; i <= radius; ++i) hw[i] = -1;
    int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
    while (dx >= dy) {
        if (dx > hw[dy]) hw[dy] = dx;
        if (dy > hw[dx]) hw[dx] = dy;
        dy++;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
}

// Host: the geometry and disc half-widths of a sweep over W x H images at cell size cs.
inline void init_base(SweepBase& B, int W, int H, int cs, const int32_t* kp_off, const float2* kps) {
    B.w = W; B.h = H; B.cs = cs; B.nwc = W / cs; B.nhc = H / cs; B.radius = cs / 4;
    circle_halfwidths(B.radius, B.hw);
    B.kp_off = kp_off; B.kps = kps;
}

__device__ __forceinline__ void paint_row(uint32_t* bm, int wpr, int W, int H, int y, int xa, int xb) {
    if (y < 0 || y >= H) return;
    xa = max(xa, 0);
    xb = min(xb, W - 1);
    if (xa > xb) return;
    uint32_t* row = bm + (size_t)y * wpr;
    const int wa = xa >> 5, wb = xb >> 5;
    for (int wi = wa; wi <= wb; ++wi) {
        uint32_t m = 0xffffffffu;
        if (wi == wa) m &= 0xffffffffu << (xa & 31);
        if (wi == wb) m &= 0xffffffffu >> (31 - (xb & 31));
        atomicOr(row + wi, m);
    }
}

// Rows r0, r0 + dr, ... of the disc around (px, py): (lane, 32) paints a whole disc with one warp, (0, 1) with one thread.
__device__ __forceinline__ void paint_disc(const SweepBase& A, uint32_t* bm, int wpr, int px, int py, int r0, int dr) {
    for (int rI = r0; rI < 2 * A.radius + 1; rI += dr) {
        const int dy = rI - A.radius;
        const int hwv = A.hw[dy < 0 ? -dy : dy];
        paint_row(bm, wpr, A.w, A.h, py + dy, px - hwv, px + hwv);
    }
}

// The row progress counters; they exist only when more than one warp sweeps.
__device__ __forceinline__ volatile int* progress_counters(const SweepSmem& L, uint8_t* sm) {
    return reinterpret_cast<volatile int*>(sm + L.progress);
}

// Block-wide: clears the bitmap, the progress counters and the occupancy grid, then marks the cells of frame fr's existing
// keypoints occupied and paints their discs (feature_extractor.cpp:316-319, 471-474), one thread per keypoint (painting
// commutes: atomicOr).  Ends with a barrier.
__device__ __forceinline__ void init_mask(const SweepBase& A, const SweepSmem& L, uint8_t* sm, int fr) {
    const int tid = threadIdx.x, nthreads = blockDim.x;
    uint32_t* bm = reinterpret_cast<uint32_t*>(sm);
    for (int i = tid; i < A.h * L.wpr; i += nthreads) bm[i] = 0;
    volatile int* progress = progress_counters(L, sm);
    if (nthreads > 32)
        for (int i = tid; i < A.nhc; i += nthreads) progress[i] = 0;
    uint8_t* occ = sm + L.occ;
    const int nocc = (A.nhc + 1) * (A.nwc + 1);
    for (int i = tid; i < nocc; i += nthreads) occ[i] = 0;
    __syncthreads();
    if (A.kp_off) {
        const int k0 = A.kp_off[fr], k1 = A.kp_off[fr + 1];
        for (int k = k0 + tid; k < k1; k += nthreads) {
            const float2 px = A.kps[k];
            const int rr = (int)(px.y / (float)A.cs), cc = (int)(px.x / (float)A.cs);
            if (rr >= 0 && rr <= A.nhc && cc >= 0 && cc <= A.nwc) occ[rr * (A.nwc + 1) + cc] = 1;
            paint_disc(A, bm, L.wpr, __float2int_rn(px.x), __float2int_rn(px.y), 0, 1);
        }
    }
    __syncthreads();
}

// Before cell (r, c): wait until row r-1 has finished cell c+1 (or its last cell).
__device__ __forceinline__ void wave_wait(volatile int* progress, int nwarps, int r, int c, int nwc) {
    if (nwarps > 1 && r > 0) {
        const int need = min(c + 2, nwc);
        while (progress[r - 1] < need) __nanosleep(40);   // yield the issue slots to the rows that are working
        __threadfence_block();
    }
}

// After cell (r, c) and its disc: publish it to row r+1.
__device__ __forceinline__ void wave_publish(volatile int* progress, int nwarps, int r, int c, int lane) {
    if (nwarps > 1) {
        __threadfence_block();                             // discs before the counter
        __syncwarp();
        if (lane == 0) progress[r] = c + 1;
    }
}

}  // namespace gsweep

// Host-side pieces the detector entry points share.

// cornerSubPix stage S on integer points (frontend_fast.cu); slots holding (-1, -1) stay empty.  d_iters: NULL, or the
// iterations each point took.
ov2_status ov2_subpix_launch(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int max_per_frame, const int2* d_int,
                             float2* d_out, int do_subpix, int32_t* d_iters);

// Device pointers of the arguments ov2_grid_fast and ov2_detect_single_scale share.
template <class State>
struct DetectArgs {
    const int32_t* kp_off = nullptr;   // NULL: no existing keypoints
    const float2* kps = nullptr;
    State* state = nullptr;            // per-frame in/out state (FAST threshold, single-scale quality)
    float2* out = nullptr;             // [count][max_per_frame] refined points
    int32_t* cnt = nullptr;            // [count]
    int2* ints = nullptr;              // [count][max_per_frame] integer points: the caller's out_pts_int or scratch
};

// Stages the shared arguments of a detector call (`what` names it in errors).  The number of existing keypoints is
// offsets[count], read back first when the offsets are on the device.
template <class State>
ov2_status stage_detect_args(ov2_ctx* ctx, const char* what, int count, int max_per_frame, const int32_t* curkp_offsets,
                             const float* curkps, State* state_inout, float* out_pts, int32_t* out_counts, int32_t* out_pts_int,
                             DetectArgs<State>* D) {
    ov2_status st;
    if (curkp_offsets) {
        if ((st = ov2_stage_in(ctx, curkp_offsets, (size_t)(count + 1), D->kp_off)) != OV2_OK) return st;
        int nkp_total = 0;
        if (ov2_is_device_ptr(curkp_offsets)) {
            OV2_CUDA(ctx, cudaMemcpyAsync(&nkp_total, curkp_offsets + count, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
            OV2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        } else {
            nkp_total = curkp_offsets[count];
        }
        if (nkp_total > 0) {
            if (!curkps) return ov2_fail(ctx, OV2_ERR_INVALID, (std::string(what) + ": curkps is NULL").c_str());
            if ((st = ov2_stage_in(ctx, curkps, (size_t)nkp_total, D->kps)) != OV2_OK) return st;
        }
    }
    if ((st = ov2_stage_out(ctx, state_inout, (size_t)count, D->state, true)) != OV2_OK) return st;
    const size_t slots = (size_t)count * max_per_frame;
    if ((st = ov2_stage_out(ctx, out_pts, slots, D->out)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, out_counts, (size_t)count, D->cnt)) != OV2_OK) return st;
    return out_pts_int ? ov2_stage_out(ctx, out_pts_int, slots, D->ints) : ov2_scratch(ctx, slots, D->ints);
}
