// MapManager::stereoMatching (/root/reference/src/map_manager.cpp:367-611) for a batch of keyframes, composed from the row
// search (ov2_line_min_sad, frontend_sad.cu) and the fbKltTracking entry point (ov2_fb_klt, frontend_klt.cu) without a host
// synchronisation between its steps:
//
//   stereo_prior_kernel   the prior of every keypoint (:396-489): a 3-D keypoint's map point projected into the right image
//                         (Tcw, then Trl, then the right camera, cam_project.cuh), or - other rigs - the inverse-distance
//                         weighted depth of the 3-D neighbours of Frame::getSurroundingKeypoints pushed along the bearing.
//                         A prior inside the right image makes the keypoint a guided one (pass-1 slot); a 3-D keypoint
//                         without a map point is dropped; the rest are blind, and on rectified rigs get a row-search slot.
//   ov2_line_min_sad      rectified rigs: the row search of all blind keypoints on level nklt_pyr_lvl, window 7, leftwards.
//   ov2_fb_klt            pass 1 over all n slots at depth 1 (:498-542).
//   stereo_retry_kernel   the pass-2 slots: blind keypoints from px, or from the accepted row-search column (:431-435), and
//                         failed guided keypoints from their pass-1 forward result (:531-535).
//   ov2_fb_klt            pass 2 over all n slots at depth nklt_pyr_lvl (:545-576); it writes the right pixels in place.
//   stereo_gate_kernel    the epipolar test of every track (:583-603): the right pixel undistorted, then the row difference
//                         (rectified: y becomes the left keypoint's undistorted y) or the Sampson distance, at most 2.
//
// Non-members of a launch are empty slots (x = -1), which the row search and the tracker skip at no cost.  The three kernels
// run one CTA of SM_THREADS threads per keyframe, each thread striding over the keyframe's keypoints, so a keyframe's count
// needs no atomics.  With device arrays the only copies are the host offset tables, and the call returns without waiting.
#include "ov2_common.cuh"
#include "cam_project.cuh"

namespace {

constexpr int SM_THREADS = 256;
constexpr int SAD_WIN = 7;                 // map_manager.cpp:378

struct SmArgs {
    int count, first, rectified;
    float up, down;                        // uppyrcoef, downpyrcoef (:380-381)
    const int32_t* offsets;                // [count + 1]
    const double* Tcw;                     // [count][12]
    const double* K;                       // [count][4], right camera
    const double* dist;                    // [count][5] or null
    const double* Trl;                     // [count][12]
    const double* Frl;                     // [count][9] (other rigs)
    const int32_t* img_wh;                 // [count][2], right image
    const int32_t* cell_offsets;           // [count + 1] (other rigs)
    const int32_t* grid;                   // [count][2] ncellsize, nbwcells (other rigs)
    const int32_t* cell_ptr;               // [cells + 1] (other rigs)
    const int32_t* cell_kps;               // [n] (other rigs)
    const float2* px;
    const float2* unpx;
    const double* bv;                      // [n][3]
    const uint8_t* is3d;
    const uint8_t* has_mp;
    const double* wpt;                     // [n][3]
    // slot arrays (device scratch) and the outputs
    int32_t* frame_idx;
    float2* kp1; float2* pri1; uint8_t* st1;
    float2* sadpt; float* xprior; float* l1err;
    float2* kp2; uint8_t* st2;
    float2* right; uint8_t* stereo; uint8_t* pass; int32_t* nstereo;
};

__device__ __forceinline__ bool member(const SmArgs& A, int i, float2 px) {
    return px.x >= 0.f && !(A.is3d[i] && !A.has_mp[i]);
}

// The depth prior of keypoint i (map_manager.cpp:438-471): the keypoints of the 2 x 2 cells up and to the left of its cell
// (Frame::getSurroundingKeypoints, src/frame.cpp:594-622: cells in loop order, then list order, the keypoint itself
// skipped), those with a map point weighted by 1 / cv::norm(unpx_j - unpx_i) (float difference, double sum of squares).
// The reference reads vgridkps_.at(idx) for idx <= size and throws at idx == size; here that cell is skipped too.
// Returns false when no neighbour has a map point; equal unpx give inf / inf = NaN, which no image contains.
__device__ bool neighbour_depth(const SmArgs& A, int f, int i, int o0, int o1, double& depth) {
    const int ncs = A.grid[2 * f], nbw = A.grid[2 * f + 1];
    const int c0 = A.cell_offsets[f], ncells = A.cell_offsets[f + 1] - c0;
    const float2 p = A.px[i], u = A.unpx[i];
    const int rk = (int)floorf(__fdiv_rn(p.y, (float)ncs)), ck = (int)floorf(__fdiv_rn(p.x, (float)ncs));
    const double* T = A.Tcw + 12 * (size_t)f;
    double zsum = 0., wsum = 0.;
    bool any = false;
    for (int r = rk - 1; r < rk + 1; ++r)
        for (int c = ck - 1; c < ck + 1; ++c) {
            const int idx = r * nbw + c;
            if (r < 0 || c < 0 || idx >= ncells) continue;
            const int b = max(A.cell_ptr[c0 + idx], o0), e = min(A.cell_ptr[c0 + idx + 1], o1);
            for (int q = b; q < e; ++q) {
                const int j = A.cell_kps[q];
                if (j == i || j < o0 || j >= o1 || !A.is3d[j] || !A.has_mp[j]) continue;
                const float dx = A.unpx[j].x - u.x, dy = A.unpx[j].y - u.y;
                const double coef = 1. / sqrt((double)dx * (double)dx + (double)dy * (double)dy);
                const double w[3] = {A.wpt[3 * (size_t)j], A.wpt[3 * (size_t)j + 1], A.wpt[3 * (size_t)j + 2]};
                double X, Y, Z;
                transform(T, w, X, Y, Z);
                wsum += coef;
                zsum += coef * Z;
                any = true;
            }
        }
    depth = zsum / wsum;
    return any;
}

// Launch: grid = count, block = SM_THREADS; keypoint i of keyframe f is visited by thread (i - offsets[f]) % SM_THREADS.
__global__ void __launch_bounds__(SM_THREADS) stereo_prior_kernel(SmArgs A) {
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    const double* T = A.Tcw + 12 * (size_t)f;
    const double* Trl = A.Trl + 12 * (size_t)f;
    const int img_w = A.img_wh[2 * f], img_h = A.img_wh[2 * f + 1];
    for (int i = o0 + threadIdx.x; i < o1; i += SM_THREADS) {
        const float2 px = A.px[i];
        const bool in = member(A, i, px);
        bool guided = false;
        float2 proj = px;
        if (in && A.is3d[i]) {                         // Frame::projWorldToRightImageDist (src/frame.cpp:835-838)
            const double w[3] = {A.wpt[3 * (size_t)i], A.wpt[3 * (size_t)i + 1], A.wpt[3 * (size_t)i + 2]};
            double c[3], X, Y, Z;
            transform(T, w, c[0], c[1], c[2]);
            transform(Trl, c, X, Y, Z);
            proj = project_dist(cam, X, Y, Z);
            guided = in_image(proj, img_w, img_h);
        }
        if (in && !guided && !A.rectified) {
            double depth;
            if (neighbour_depth(A, f, i, o0, o1, depth)) {   // Frame::projCamToRightImageDist(mean_z * bv / bv.z)
                const double* b = A.bv + 3 * (size_t)i;
                const double c[3] = {depth * (b[0] / b[2]), depth * (b[1] / b[2]), depth * (b[2] / b[2])};
                double X, Y, Z;
                transform(Trl, c, X, Y, Z);
                proj = project_dist(cam, X, Y, Z);
                guided = in_image(proj, img_w, img_h);
            }
        }
        A.frame_idx[i] = A.first + f;
        A.kp1[i] = guided ? px : make_float2(-1.f, -1.f);
        A.pri1[i] = guided ? proj : px;
        if (A.rectified)
            A.sadpt[i] = in && !guided ? make_float2(px.x * A.down, px.y * A.down) : make_float2(-1.f, -1.f);
    }
}

// Launch: as stereo_prior_kernel.
__global__ void __launch_bounds__(SM_THREADS) stereo_retry_kernel(SmArgs A) {
    const int f = blockIdx.x;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += SM_THREADS) {
        const float2 px = A.px[i];
        const bool guided = A.kp1[i].x >= 0.f;
        if (guided && A.st1[i]) {
            // tracked with its prior: an empty slot of pass 2 that keeps the pass-1 result
            A.kp2[i] = make_float2(-1.f, -1.f);
            A.right[i] = A.pri1[i];
            A.pass[i] = 1;
        } else if (member(A, i, px)) {
            float2 pri = guided ? A.pri1[i] : px;
            if (!guided && A.rectified) {
                const float x = A.xprior[i] * A.up;
                if (x >= 0.f && x <= px.x) pri.x = x;
            }
            A.kp2[i] = px;
            A.right[i] = pri;
            A.pass[i] = 2;
        } else {
            A.kp2[i] = make_float2(-1.f, -1.f);
            A.right[i] = px;
            A.pass[i] = 0;
        }
    }
}

// MultiViewGeometry::computeSampsonDistance (src/multi_view_geometry.cpp:798-821): the products in double (rows summed left
// to right, r^T F formed before the product with l), every result rounded to float, the rest in float.
__device__ __forceinline__ float sampson(const double* F, float2 l, float2 r) {
    const double lx = l.x, ly = l.y, rx = r.x, ry = r.y;
    const double t0 = rx * F[0] + ry * F[3] + F[6];          // r^T F = (F^T r)^T
    const double t1 = rx * F[1] + ry * F[4] + F[7];
    const double t2 = rx * F[2] + ry * F[5] + F[8];
    float num = (float)(t0 * lx + t1 * ly + t2);
    num = num * num;
    const float x1 = (float)t0, y1 = (float)t1;
    const float x2 = (float)(F[0] * lx + F[1] * ly + F[2]);
    const float y2 = (float)(F[3] * lx + F[4] * ly + F[5]);
    const float den = x1 * x1 + y1 * y1 + x2 * x2 + y2 * y2;
    return __fsqrt_rn(__fdiv_rn(num, den));
}

// Launch: as stereo_prior_kernel.  The keyframe's count is a CTA reduction of per-thread counts (integers: order independent).
__global__ void __launch_bounds__(SM_THREADS) stereo_gate_kernel(SmArgs A) {
    __shared__ int s_n[SM_THREADS / 32];
    const int f = blockIdx.x;
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    int nst = 0;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += SM_THREADS) {
        const int pass = A.pass[i];
        bool ok = pass == 1 || (pass == 2 && A.st2[i]);
        if (ok) {
            float2 r = A.right[i];
            const float2 lun = A.unpx[i], run = undistort_point(cam, r.x, r.y);
            float err;
            if (A.rectified) {
                err = fabsf(lun.y - run.y);
                r.y = lun.y;
                A.right[i] = r;
            } else {
                err = sampson(A.Frl + 9 * (size_t)f, lun, run);
            }
            ok = err <= 2.f;
        }
        A.stereo[i] = ok;
        nst += ok;
    }
    nst = __reduce_add_sync(0xffffffffu, nst);
    if ((threadIdx.x & 31) == 0) s_n[threadIdx.x >> 5] = nst;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int k = 0; k < SM_THREADS / 32; ++k) t += s_n[k];
        A.nstereo[f] = t;
    }
}

struct Inputs {
    const int32_t* offsets; const double* Tcw; const double* K; const double* dist; const double* Trl; const double* Frl;
    const int32_t* img_wh; const int32_t* cell_offsets; const int32_t* grid; const int32_t* cell_ptr; const int32_t* cell_kps;
    const float* px; const float* unpx; const double* bv; const uint8_t* is3d; const uint8_t* has_mp; const double* wpt;
    float* right_out; uint8_t* stereo_out; uint8_t* pass_out; int32_t* nstereo_out;
};

ov2_status enqueue(ov2_ctx* ctx, const ov2_pyr* left, const ov2_pyr* right, const ov2_klt_params* prm, int n, int nklt_pyr_lvl,
                   SmArgs& A, const Inputs& in) {
    const size_t nn = (size_t)n, nc = (size_t)A.count;
    ov2_status st;
    const void* d = nullptr;
    void* o = nullptr;
#define IN(ptr, bytes, field, type) do { if ((st = ov2_stage_in(ctx, ptr, bytes, &d)) != OV2_OK) return st; A.field = (const type*)d; } while (0)
#define OUT(ptr, bytes, field, type) do { if ((st = ov2_stage_out(ctx, ptr, bytes, &o)) != OV2_OK) return st; A.field = (type*)o; } while (0)
#define SCRATCH(bytes, field, type) do { if ((st = ov2_scratch(ctx, bytes, &o)) != OV2_OK) return st; A.field = (type*)o; } while (0)
    IN(in.offsets, sizeof(int32_t) * (nc + 1), offsets, int32_t);
    IN(in.Tcw, sizeof(double) * 12 * nc, Tcw, double);
    IN(in.K, sizeof(double) * 4 * nc, K, double);
    IN(in.dist, sizeof(double) * 5 * nc, dist, double);
    IN(in.Trl, sizeof(double) * 12 * nc, Trl, double);
    IN(in.img_wh, sizeof(int32_t) * 2 * nc, img_wh, int32_t);
    OUT(in.nstereo_out, sizeof(int32_t) * nc, nstereo, int32_t);
    if (!A.rectified) {
        IN(in.Frl, sizeof(double) * 9 * nc, Frl, double);
        IN(in.cell_offsets, sizeof(int32_t) * (nc + 1), cell_offsets, int32_t);
        IN(in.grid, sizeof(int32_t) * 2 * nc, grid, int32_t);
        IN(in.cell_ptr, sizeof(int32_t) * ((size_t)in.cell_offsets[A.count] + 1), cell_ptr, int32_t);
    }
    if (n > 0) {
        IN(in.px, sizeof(float2) * nn, px, float2);
        IN(in.unpx, sizeof(float2) * nn, unpx, float2);
        IN(in.is3d, nn, is3d, uint8_t);
        IN(in.has_mp, nn, has_mp, uint8_t);
        IN(in.wpt, sizeof(double) * 3 * nn, wpt, double);
        OUT(in.right_out, sizeof(float2) * nn, right, float2);
        OUT(in.stereo_out, nn, stereo, uint8_t);
        OUT(in.pass_out, nn, pass, uint8_t);
        SCRATCH(sizeof(int32_t) * nn, frame_idx, int32_t);
        SCRATCH(sizeof(float2) * nn, kp1, float2);
        SCRATCH(sizeof(float2) * nn, pri1, float2);
        SCRATCH(nn, st1, uint8_t);
        SCRATCH(sizeof(float2) * nn, kp2, float2);
        SCRATCH(nn, st2, uint8_t);
        if (A.rectified) {
            SCRATCH(sizeof(float2) * nn, sadpt, float2);
            SCRATCH(sizeof(float) * nn, xprior, float);
            SCRATCH(sizeof(float) * nn, l1err, float);
        } else {
            IN(in.bv, sizeof(double) * 3 * nn, bv, double);
            IN(in.cell_kps, sizeof(int32_t) * nn, cell_kps, int32_t);
        }
    }
#undef IN
#undef OUT
#undef SCRATCH
    OV2_LAUNCH(ctx, "stereo_prior_kernel", stereo_prior_kernel<<<A.count, SM_THREADS, 0, ctx->stream>>>(A));
    if (A.rectified && (st = ov2_line_min_sad(ctx, left, right, nklt_pyr_lvl, n, A.frame_idx, 0, 0, (const float*)A.sadpt, SAD_WIN,
                                              1, A.xprior, A.l1err)) != OV2_OK)
        return st;
    if ((st = ov2_fb_klt(ctx, left, right, prm, n, A.frame_idx, 0, 0, nullptr, 1, (const float*)A.kp1, (float*)A.pri1, A.st1)) != OV2_OK)
        return st;
    OV2_LAUNCH(ctx, "stereo_retry_kernel", stereo_retry_kernel<<<A.count, SM_THREADS, 0, ctx->stream>>>(A));
    if ((st = ov2_fb_klt(ctx, left, right, prm, n, A.frame_idx, 0, 0, nullptr, nklt_pyr_lvl, (const float*)A.kp2, (float*)A.right,
                         A.st2)) != OV2_OK)
        return st;
    OV2_LAUNCH(ctx, "stereo_gate_kernel", stereo_gate_kernel<<<A.count, SM_THREADS, 0, ctx->stream>>>(A));
    return OV2_OK;
}

// a host table that starts at 0 and never decreases
bool ascending(const int32_t* t, int count) {
    if (t[0] != 0) return false;
    for (int k = 0; k < count; ++k)
        if (t[k + 1] < t[k]) return false;
    return true;
}

}  // namespace

extern "C" ov2_status ov2_stereo_matching(ov2_ctx* ctx, const ov2_pyr* left, const ov2_pyr* right, const ov2_klt_params* prm,
                                          int first, int count, const int32_t* offsets, const double* Tcw, const double* K,
                                          const double* dist, const double* Trl, const double* Frl, const int32_t* img_wh,
                                          const int32_t* cell_offsets, const int32_t* grid, const int32_t* cell_ptr,
                                          const int32_t* cell_kps, const float* px, const float* unpx, const double* bv,
                                          const uint8_t* is3d, const uint8_t* has_mp, const double* wpt, int rectified,
                                          int nklt_pyr_lvl, float* right_out, uint8_t* stereo_out, uint8_t* pass_out,
                                          int32_t* nstereo_out) {
    if (!ctx || !left || !right || !prm || count < 0 || nklt_pyr_lvl < 0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: bad arguments");
    if (count == 0) return OV2_OK;
    if (!offsets || !Tcw || !K || !Trl || !img_wh || !nstereo_out || (!rectified && (!Frl || !cell_offsets || !grid || !cell_ptr)))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: null array");
    if (ov2_is_device_ptr(offsets) || (!rectified && ov2_is_device_ptr(cell_offsets)))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: offsets and cell_offsets must be host pointers");
    // every keyframe's CTA reads offsets[f] .. offsets[f + 1] of arrays sized offsets[count], and its cells likewise
    if (!ascending(offsets, count) || (!rectified && !ascending(cell_offsets, count)))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: offsets must start at 0 and be ascending");
    const int n = offsets[count];
    if (n > 0 && (!px || !unpx || !is3d || !has_mp || !wpt || !right_out || !stereo_out || !pass_out || (!rectified && (!bv || !cell_kps))))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: null array");
    if (first < 0 || first + count > left->batch || first + count > right->batch)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: more keyframes than pyramid slots");
    if (prm->win < 3 || prm->win > 31) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: nwinsize must be 3 .. 31");
    if (left->nlev != right->nlev || left->w[0] != right->w[0] || left->h[0] != right->h[0] || !left->l0 || !right->l0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: pyramids not built / mismatched");
    // the row search reads vleftpyr.at(2 * nklt_pyr_lvl) (map_manager.cpp:429); ov2_line_min_sad serves levels 0 .. 3
    if (rectified && (nklt_pyr_lvl >= left->nlev || nklt_pyr_lvl > 3))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: the pyramids have no level nklt_pyr_lvl for the row search");
    // batch mode inside (unless the caller has a batch open): the row search's and the trackers' calls only enqueue, scratch
    // survives between them, and host outputs come back with one synchronisation at the end
    const bool own_batch = !ctx->batch;
    ov2_status st = own_batch ? ov2_batch_begin(ctx) : ov2_begin(ctx);
    if (st != OV2_OK) return st;
    SmArgs A = {};
    A.count = count;
    A.first = first;
    A.rectified = rectified ? 1 : 0;
    A.up = (float)std::pow(2., nklt_pyr_lvl);
    A.down = (float)(1. / A.up);
    const Inputs in = {offsets, Tcw, K, dist, Trl, Frl, img_wh, cell_offsets, grid, cell_ptr, cell_kps, px, unpx, bv, is3d, has_mp,
                       wpt, right_out, stereo_out, pass_out, nstereo_out};
    st = enqueue(ctx, left, right, prm, n, nklt_pyr_lvl, A, in);
    if (!own_batch) return st;
    ctx->batch = false;
    if (st != OV2_OK) {
        ctx->pending.clear();
        return st;
    }
    if (ctx->pending.empty()) return OV2_OK;      // device outputs only: enqueued, as every other call with device pointers
    if ((st = ov2_batch_flush_outputs(ctx)) != OV2_OK) return st;
    return ov2_wait_stream(ctx);
}
