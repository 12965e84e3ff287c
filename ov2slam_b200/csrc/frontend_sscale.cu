// D ("next" row, SURVEY.md 8f-1): FeatureExtractor::detectSingleScale
// (/root/reference/src/feature_extractor.cpp:288-440): per cell GaussianBlur 3x3 -> cornerMinEigenVal(3, 3)
// -> arg-max of (response * mask) twice with the disc mask of detectGridFAST, second detections fill the
// cells that stayed empty, adaptive dmaxquality_ (:418-423), cornerSubPix (:424-436, stage S).
//
// OpenCV semantics implemented here are the ones oracle/image_ref.py pins against cv2 4.13
// (blur3_cell_ref / min_eigen_ref / _first_max; tests/test_oracle_image.py):
//   * the blur of a cell SUB-MATRIX takes its border pixels from the parent image and rounds S/16
//     half-to-even in the first 16*floor(cs/16) columns, half-up in the rest;
//   * Sobel / products / eigenvalue in float32 with OpenCV's operation order (every float operation below
//     is an explicit __f*_rn intrinsic: nothing is contracted), 3x3 sums exact (double) then one rounding;
//   * arg-max = first maximum in row-major order; the sequential cell order is the semantics (the
//     reference's parallel_for_ body races on the mask).
//
// Two kernels: ss_response_kernel (one CTA per cell and frame, everything in shared memory, response map
// to HBM: 4 B/pixel written once, read at most twice) and ss_sweep_kernel (one CTA per frame, one warp per cell row in a
// wavefront that reproduces the sequential cell order, 1 bit/pixel mask in shared memory).
#include "ov2_common.cuh"
#include "grid_sweep.cuh"
#include "sscale_math.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int SS_MAX_CELL = 64;

struct RespArgs {
    const uint8_t* img; int w, h, pitch; long long fstride;
    int first, cs, nwc, nhc;
    float* resp;            // [count][ncells][cs*cs]
    float2* cellmax;        // [count][ncells]: (first maximum of the cell's response, its row-major index as int bits)
};

__global__ void __launch_bounds__(256) ss_response_kernel(RespArgs A) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int cs = A.cs, cell = blockIdx.x, fr = blockIdx.y;
    const int r = cell / A.nwc, c = cell - r * A.nwc;
    const int x0 = c * cs, y0 = r * cs;
    if (!(x0 + cs < A.w - 1 && y0 + cs < A.h - 1)) return;      // never searched (feature_extractor.cpp:346)
    const int rw = cs + 2;
    uint8_t* raw = smem;                                          // (cs+2)^2: cell + 1-px halo from the PARENT image
    uint8_t* bl = raw + sscale::raw_bytes(cs);                    // cs^2 blurred
    double* cov = reinterpret_cast<double*>(bl + sscale::blur_bytes(cs));   // Sobel products [pixel][xx, xy, yy]
    const uint8_t* img = A.img + A.fstride * (A.first + fr);
    {   // staging: a warp per tile row, a lane per column - the reflected column is formed once per lane, the row once per warp
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
        for (int xx = lane; xx < rw; xx += 32) {
            const int gx = sscale::refl(x0 - 1 + xx, A.w);
            for (int yy = warp; yy < rw; yy += nwarp) {
                const int gy = sscale::refl(y0 - 1 + yy, A.h);
                raw[yy * rw + xx] = __ldg(img + (size_t)gy * A.pitch + gx);
            }
        }
    }
    __syncthreads();
    sscale::phase_blur(threadIdx.x, blockDim.x, raw, bl, cs);
    __syncthreads();
    sscale::phase_cov(threadIdx.x, blockDim.x, bl, cov, cs);
    __syncthreads();
    float* out = A.resp + ((size_t)fr * (A.nwc * A.nhc) + cell) * (size_t)(cs * cs);
    // first maximum (row-major) of the unmasked response, tracked while the responses are written: lets the sweep skip its
    // first arg-max scan whenever that pixel is not masked (the usual case)
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    sscale::phase_response(threadIdx.x, blockDim.x, cov, out, cs, bv, bi);
    __shared__ float s_v[8];
    __shared__ int s_i[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(FULL, bv, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
            if (s_v[k] > bv || (s_v[k] == bv && s_i[k] < bi)) { bv = s_v[k]; bi = s_i[k]; }
        A.cellmax[(size_t)fr * (A.nwc * A.nhc) + cell] = make_float2(bv, __int_as_float(bi));
    }
}

struct SweepArgs : gsweep::SweepBase {
    int max_per_frame;
    int roi_x, roi_y, roi_w, roi_h;
    const float* resp;               // [count][ncells][cs*cs]
    const float2* cellmax;           // [count][ncells] first maximum per cell (value, index bits)
    double* quality;                 // in/out per frame
    int2* out_int;                   // [count][max_per_frame]
    int32_t* out_n;                  // [count]
};

constexpr int SWEEP_MAX_WARPS = 32;

// First maximum (row-major) of resp * mask over one cell by ONE warp; every lane returns the same (value, index).
__device__ __forceinline__ void cell_argmax_warp(const float* __restrict__ resp, const uint32_t* bm, int wpr, int x0, int y0, int cs,
                                                 int lane, float& best_v, int& best_i) {
    const int npx = cs * cs;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    int yy = lane / cs, xx = lane - yy * cs;
    const int sy = 32 / cs, sx = 32 - sy * cs;
    for (int i = lane; i < npx; i += 32) {
        const int gx = x0 + xx, gy = y0 + yy;
        const bool masked = (bm[(size_t)gy * wpr + (gx >> 5)] >> (gx & 31)) & 1u;
        const float v = masked ? 0.0f : __ldg(resp + i);           // response * 0.0f compares equal to 0
        if (v > bv) { bv = v; bi = i; }                           // strict: the earliest index of this lane wins
        xx += sx; yy += sy;
        if (xx >= cs) { xx -= cs; yy++; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(FULL, bv, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    best_v = bv; best_i = bi;
}

// Shared-memory layout of ss_sweep_kernel: two detections per cell (int2, x < 0: none) between the bitmap and the counters.
__host__ __device__ inline gsweep::SweepSmem ss_sweep_smem(int w, int h, int nwc, int nhc, int nwarps) {
    return gsweep::SweepSmem(w, h, nwc, nhc, nwarps, (gsweep::SweepSmem::off)nwc * nhc * 2 * sizeof(int2), alignof(int2));
}

// The wavefront sweep of grid_sweep.cuh, one warp per cell row.
__global__ void __launch_bounds__(SWEEP_MAX_WARPS * 32, 1) ss_sweep_kernel(SweepArgs A) {
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ int s_n;
    const int tid = threadIdx.x, fr = blockIdx.x, nthreads = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nthreads >> 5;
    const int ncells = A.nwc * A.nhc, cs = A.cs;
    const gsweep::SweepSmem L = ss_sweep_smem(A.w, A.h, A.nwc, A.nhc, nwarps);
    const int wpr = L.wpr;
    uint32_t* bm = reinterpret_cast<uint32_t*>(sm);
    int2* firstd = reinterpret_cast<int2*>(sm + L.mid);
    int2* secondd = firstd + ncells;
    volatile int* progress = gsweep::progress_counters(L, sm);
    const uint8_t* occ = sm + L.occ;
    for (int i = tid; i < ncells; i += nthreads) { firstd[i] = make_int2(-1, -1); secondd[i] = make_int2(-1, -1); }
    gsweep::init_mask(A, L, sm, fr);
    const double quality = A.quality[fr];
    const float* resp = A.resp + (size_t)fr * ncells * (size_t)(cs * cs);
    constexpr int NV = 40;                                        // register-resident cells: cs * cs <= 1280 (cs <= 35)
    const int npx = cs * cs;
    const bool in_regs = npx <= NV * 32;
    const int sy = 32 / cs, sx = 32 - sy * cs;
    for (int r = warp; r < A.nhc; r += nwarps) {
        for (int c = 0; c < A.nwc; ++c) {
            const int cell = r * A.nwc + c;
            const int x0 = c * cs, y0 = r * cs;
            const bool search = !occ[r * (A.nwc + 1) + c] && (x0 + cs < A.w - 1 && y0 + cs < A.h - 1);
            const float* rc = resp + (size_t)cell * npx;
            // the cell's responses do not depend on any other cell: fetch them (all loads in flight at once) BEFORE waiting
            // for the neighbours, so the L2 latency hides behind the wavefront dependency
            float v[NV];
            if (search && in_regs) {
#pragma unroll
                for (int q = 0; q < NV; ++q) {
                    const int i = lane + 32 * q;
                    v[q] = i < npx ? __ldg(rc + i) : -INFINITY;
                }
            }
            gsweep::wave_wait(progress, nwarps, r, c, A.nwc);
            if (search) {
                const float2 cm = A.cellmax[(size_t)fr * ncells + cell];
                for (int round = 0; round < 2; ++round) {
                    float mx; int idx;
                    bool have = false;
                    if (round == 0 && cm.x > 0.0f) {
                        // the cell's first maximum is the answer unless a disc already covers it (masked pixels count as 0 < cm.x)
                        const int ci = __float_as_int(cm.y);
                        const int qy = ci / cs, qx = ci - qy * cs;
                        const int gx = x0 + qx, gy = y0 + qy;
                        if (!((bm[(size_t)gy * wpr + (gx >> 5)] >> (gx & 31)) & 1u)) { mx = cm.x; idx = ci; have = true; }
                    }
                    if (have) {
                    } else if (in_regs) {
                        float bv = -INFINITY;
                        int bi = 0x7fffffff;
                        int yy = lane / cs, xx = lane - yy * cs;
#pragma unroll
                        for (int q = 0; q < NV; ++q) {
                            const int i = lane + 32 * q;
                            if (i < npx) {
                                const int gx = x0 + xx, gy = y0 + yy;
                                const bool masked = (bm[(size_t)gy * wpr + (gx >> 5)] >> (gx & 31)) & 1u;
                                const float val = masked ? 0.0f : v[q];          // response * 0.0f compares equal to 0
                                if (val > bv) { bv = val; bi = i; }
                                xx += sx; yy += sy;
                                if (xx >= cs) { xx -= cs; yy++; }
                            }
                        }
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) {
                            const float ov = __shfl_xor_sync(FULL, bv, o);
                            const int oi = __shfl_xor_sync(FULL, bi, o);
                            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
                        }
                        mx = bv; idx = bi;
                    } else {
                        cell_argmax_warp(rc, bm, wpr, x0, y0, cs, lane, mx, idx);
                    }
                    const int ly = idx / cs, lx = idx - ly * cs;
                    const int px = x0 + lx, py = y0 + ly;
                    if (px < A.roi_x || py < A.roi_y || px >= A.roi_x + A.roi_w || py >= A.roi_y + A.roi_h) break;   // `continue` of the cell loop
                    if ((double)mx >= quality) {
                        if (lane == 0) (round == 0 ? firstd : secondd)[cell] = make_int2(px, py);
                        gsweep::paint_disc(A, bm, wpr, px, py, lane, 32);
                        __syncwarp();
                    }
                }
            }
            gsweep::wave_publish(progress, nwarps, r, c, lane);
        }
    }
    __syncthreads();
    // assembly (feature_extractor.cpp:393-423): first detections in cell order, then second detections
    // while cells stayed empty; quality adaptation; unused slots = (-1, -1)
    int2* out = A.out_int + (size_t)fr * A.max_per_frame;
    if (tid == 0) {
        int nboccup = 0;
        for (int cell = 0; cell < ncells; ++cell) {
            const int r = cell / A.nwc, c = cell - r * A.nwc;
            nboccup += occ[r * (A.nwc + 1) + c] ? 1 : 0;
        }
        int n = 0;
        for (int cell = 0; cell < ncells; ++cell)
            if (firstd[cell].x >= 0 && n < A.max_per_frame) out[n++] = firstd[cell];
        if (n + nboccup < ncells) {
            const int nbsec = ncells - (n + nboccup);
            int k = 0;
            for (int cell = 0; cell < ncells && k < nbsec; ++cell)
                if (secondd[cell].x >= 0) {
                    if (n < A.max_per_frame) out[n++] = secondd[cell];
                    k++;
                }
        }
        double q = quality;
        if ((double)n < 0.33 * (double)(ncells - nboccup)) q /= 2.0;
        else if ((double)n > 0.9 * (double)(ncells - nboccup)) q *= 1.5;
        A.quality[fr] = q;
        A.out_n[fr] = n;
        s_n = n;
    }
    __syncthreads();
    for (int i = s_n + tid; i < A.max_per_frame; i += nthreads) out[i] = make_int2(-1, -1);
}

}  // namespace

extern "C" ov2_status ov2_detect_single_scale(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int cellsize,
                                              const int32_t* curkp_offsets, const float* curkps, const int32_t* roi_xywh,
                                              double* quality_inout, int max_per_frame, float* out_pts, int32_t* out_counts,
                                              int32_t* out_pts_int, int do_subpix) {
    if (!ctx || !pyr || !pyr->l0 || first < 0 || count <= 0 || first + count > pyr->batch || !quality_inout || !out_pts ||
        !out_counts)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_detect_single_scale: bad arguments");
    if (cellsize < 8 || cellsize > SS_MAX_CELL)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_detect_single_scale: cellsize must be in [8, 64]");
    const int W = pyr->w[0], H = pyr->h[0];
    const int nwc = W / cellsize, nhc = H / cellsize, ncells = nwc * nhc;
    if (ncells == 0 || max_per_frame < ncells)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_detect_single_scale: max_per_frame < number of cells");
    int roi[4] = {0, 0, W, H};
    if (roi_xywh) {
        if (ov2_is_device_ptr(roi_xywh)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_detect_single_scale: roi must be a host pointer");
        for (int i = 0; i < 4; ++i) roi[i] = roi_xywh[i];
    }
    const int nw = nhc < SWEEP_MAX_WARPS ? nhc : SWEEP_MAX_WARPS;       // one warp per cell row (wavefront)
    const size_t sweep_smem = ss_sweep_smem(W, H, nwc, nhc, nw).bytes;
    if (sweep_smem > gsweep::SMEM_LIMIT)
        return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_detect_single_scale: image too large for the shared-memory mask bitmap");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    DetectArgs<double> D;
    if ((st = stage_detect_args(ctx, "ov2_detect_single_scale", count, max_per_frame, curkp_offsets, curkps, quality_inout, out_pts,
                                out_counts, out_pts_int, &D)) != OV2_OK)
        return st;
    const size_t cell_px = (size_t)cellsize * cellsize;
    float* d_resp = nullptr;
    float2* d_cellmax = nullptr;
    if ((st = ov2_scratch(ctx, (size_t)count * ncells * cell_px, d_resp)) != OV2_OK) return st;
    if ((st = ov2_scratch(ctx, (size_t)count * ncells, d_cellmax)) != OV2_OK) return st;

    RespArgs RA;
    RA.img = pyr->l0; RA.w = W; RA.h = H; RA.pitch = (int)pyr->l0_pitch; RA.fstride = (long long)pyr->l0_fstride;
    RA.first = first; RA.cs = cellsize; RA.nwc = nwc; RA.nhc = nhc; RA.resp = d_resp; RA.cellmax = d_cellmax;
    {
        const size_t smem = sscale::smem_bytes(cellsize);
        if (smem > 48 * 1024)
            OV2_CUDA(ctx, cudaFuncSetAttribute(ss_response_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        OV2_LAUNCH(ctx, "ss_response_kernel", ss_response_kernel<<<dim3(ncells, count), 256, smem, ctx->stream>>>(RA));
    }
    SweepArgs SA;
    gsweep::init_base(SA, W, H, cellsize, D.kp_off, D.kps);
    SA.max_per_frame = max_per_frame;
    SA.roi_x = roi[0]; SA.roi_y = roi[1]; SA.roi_w = roi[2]; SA.roi_h = roi[3];
    SA.resp = d_resp; SA.cellmax = d_cellmax; SA.quality = D.state; SA.out_int = D.ints; SA.out_n = D.cnt;
    if (sweep_smem > 48 * 1024)
        OV2_CUDA(ctx, cudaFuncSetAttribute(ss_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sweep_smem));
    OV2_LAUNCH(ctx, "ss_sweep_kernel", ss_sweep_kernel<<<count, nw * 32, sweep_smem, ctx->stream>>>(SA));
    if ((st = ov2_subpix_launch(ctx, pyr, first, count, max_per_frame, D.ints, D.out, do_subpix, nullptr)) != OV2_OK) return st;
    return ov2_end(ctx);
}
