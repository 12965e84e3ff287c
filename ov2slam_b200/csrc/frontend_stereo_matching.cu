// MapManager::stereoMatching (/root/reference/src/map_manager.cpp:367-611) for a batch of keyframes, composed from the row
// search (ov2_line_min_sad, frontend_sad.cu) and the fbKltTracking entry point (ov2_fb_klt, frontend_klt.cu) without a host
// synchronisation between its steps:
//
//   stereo_prior_kernel   the prior of every keypoint (:396-489): a 3-D keypoint's map point projected into the right image
//                         (Tcw, then Trl, then the right camera, cam_project.cuh), or - other rigs - the inverse-distance
//                         weighted depth of the 3-D neighbours of Frame::getSurroundingKeypoints pushed along the bearing.
//                         A prior inside the right image makes the keypoint a guided one, and the kernel writes the pass-1
//                         slots; a 3-D keypoint without a map point is dropped; the rest are blind, and on rectified rigs get
//                         a row-search slot.
//   ov2_line_min_sad      rectified rigs: the row search of all blind keypoints on level nklt_pyr_lvl, window 7, leftwards.
//   ov2_fb_klt            pass 1 at depth 1 (:498-542).
//   stereo_retry_kernel   the pass-2 slots.  The members are the keypoints not dropped; blind keypoints restart from px, or
//                         from the accepted row-search column (:431-435), and failed guided keypoints from their pass-1
//                         forward result (:531-535).
//   ov2_fb_klt            pass 2 at depth nklt_pyr_lvl (:545-576); it writes the right pixels in place.
//   stereo_gate_kernel    the epipolar test of every track (:583-603): the right pixel undistorted, then the row difference
//                         (rectified: y becomes the left keypoint's undistorted y) or the Sampson distance, at most 2.
//
// Non-members of the row search are empty slots (x = -1), which it skips at no cost.  The three kernels run one CTA per
// keyframe and write the slots by the shared two-pass protocol (two_pass.cuh).  With device arrays the only copies are the
// host offset tables, and the call returns without waiting.
#include "ov2_common.cuh"
#include "cam_project.cuh"
#include "two_pass.cuh"

namespace {

using namespace two_pass;

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
    TwoPass tp;
    float2* sadpt; float* xprior; float* l1err;   // row-search slots and results (rectified rigs)
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

// Launch: grid = count, block = THREADS; keypoint i of keyframe f is visited by thread (i - offsets[f]) % THREADS.
__global__ void __launch_bounds__(THREADS) stereo_prior_kernel(SmArgs A) {
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    const double* T = A.Tcw + 12 * (size_t)f;
    const double* Trl = A.Trl + 12 * (size_t)f;
    const int img_w = A.img_wh[2 * f], img_h = A.img_wh[2 * f + 1];
    for (int i = o0 + threadIdx.x; i < o1; i += THREADS) {
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
        A.tp.set_pass1(i, A.first + f, px, guided, proj);
        if (A.rectified)
            A.sadpt[i] = in && !guided ? make_float2(px.x * A.down, px.y * A.down) : make_float2(-1.f, -1.f);
    }
}

// Launch: as stereo_prior_kernel.
__global__ void __launch_bounds__(THREADS) stereo_retry_kernel(SmArgs A) {
    const int f = blockIdx.x;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += THREADS) {
        const float2 px = A.px[i];
        const bool guided = A.tp.kp1[i].x >= 0.f;
        float2 restart = guided ? A.tp.pri1[i] : px;
        if (!guided && A.rectified) {
            const float x = A.xprior[i] * A.up;
            if (x >= 0.f && x <= px.x) restart.x = x;
        }
        // every guided keypoint is a member: its test needs no loads
        A.tp.set_pass2(i, px, guided || member(A, i, px), restart, A.right, A.pass);
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

// Launch: as stereo_prior_kernel.
__global__ void __launch_bounds__(THREADS) stereo_gate_kernel(SmArgs A) {
    __shared__ int s_n[THREADS / 32];
    const int f = blockIdx.x;
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    int nst = 0;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += THREADS) {
        const int pass = A.pass[i];
        bool ok = pass == 1 || (pass == 2 && A.tp.st2[i]);
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
    nst = cta_sum(nst, s_n);
    if (threadIdx.x == 0) A.nstereo[f] = nst;
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
    // every keyframe's CTA reads offsets[f] .. offsets[f + 1] of arrays sized offsets[count], and its cells likewise
    const ov2_offsets_check oc = ov2_check_offsets(offsets, count);
    const ov2_offsets_check cc = rectified ? OV2_OFFSETS_OK : ov2_check_offsets(cell_offsets, count);
    if (oc == OV2_OFFSETS_ON_DEVICE || cc == OV2_OFFSETS_ON_DEVICE)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: offsets and cell_offsets must be host pointers");
    if (oc != OV2_OFFSETS_OK || cc != OV2_OFFSETS_OK)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: offsets must start at 0 and be ascending");
    const int n = offsets[count];
    if (n > 0 && (!px || !unpx || !is3d || !has_mp || !wpt || !right_out || !stereo_out || !pass_out || (!rectified && (!bv || !cell_kps))))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: null array");
    if (first < 0 || first + count > left->batch || first + count > right->batch)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: more keyframes than pyramid slots");
    if (prm->win < 3 || prm->win > 31) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: nwinsize must be 3 .. 31");
    if (!ov2_pyr_pair_ok(left, right)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: pyramids not built / mismatched");
    // the row search reads vleftpyr.at(2 * nklt_pyr_lvl) (map_manager.cpp:429); ov2_line_min_sad serves levels 0 .. 3
    if (rectified && (nklt_pyr_lvl >= left->nlev || nklt_pyr_lvl > 3))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_stereo_matching: the pyramids have no level nklt_pyr_lvl for the row search");
    return ov2_in_batch(ctx, [&]() -> ov2_status {
        const size_t nn = (size_t)n, nc = (size_t)count;
        SmArgs A = {};
        A.count = count;
        A.first = first;
        A.rectified = rectified ? 1 : 0;
        A.up = (float)std::pow(2., nklt_pyr_lvl);
        A.down = (float)(1. / A.up);
        ov2_status st;
        if ((st = ov2_stage_in(ctx, offsets, nc + 1, A.offsets)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, Tcw, 12 * nc, A.Tcw)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, K, 4 * nc, A.K)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, dist, 5 * nc, A.dist)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, Trl, 12 * nc, A.Trl)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, img_wh, 2 * nc, A.img_wh)) != OV2_OK) return st;
        if ((st = ov2_stage_out(ctx, nstereo_out, nc, A.nstereo)) != OV2_OK) return st;
        if (!rectified) {
            if ((st = ov2_stage_in(ctx, Frl, 9 * nc, A.Frl)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, cell_offsets, nc + 1, A.cell_offsets)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, grid, 2 * nc, A.grid)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, cell_ptr, (size_t)cell_offsets[count] + 1, A.cell_ptr)) != OV2_OK) return st;
        }
        if (n > 0) {
            if ((st = ov2_stage_in(ctx, px, nn, A.px)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, unpx, nn, A.unpx)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, is3d, nn, A.is3d)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, has_mp, nn, A.has_mp)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, wpt, 3 * nn, A.wpt)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, right_out, nn, A.right)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, stereo_out, nn, A.stereo)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, pass_out, nn, A.pass)) != OV2_OK) return st;
            if ((st = A.tp.stage(ctx, nn)) != OV2_OK) return st;
            if (rectified) {
                if ((st = ov2_scratch(ctx, nn, A.sadpt)) != OV2_OK) return st;
                if ((st = ov2_scratch(ctx, nn, A.xprior)) != OV2_OK) return st;
                if ((st = ov2_scratch(ctx, nn, A.l1err)) != OV2_OK) return st;
            } else {
                if ((st = ov2_stage_in(ctx, bv, 3 * nn, A.bv)) != OV2_OK) return st;
                if ((st = ov2_stage_in(ctx, cell_kps, nn, A.cell_kps)) != OV2_OK) return st;
            }
        }
        OV2_LAUNCH(ctx, "stereo_prior_kernel", stereo_prior_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        if (rectified && (st = ov2_line_min_sad(ctx, left, right, nklt_pyr_lvl, n, A.tp.frame_idx, 0, 0, (const float*)A.sadpt,
                                                SAD_WIN, 1, A.xprior, A.l1err)) != OV2_OK)
            return st;
        if ((st = A.tp.pass1(ctx, left, right, prm, n)) != OV2_OK) return st;
        OV2_LAUNCH(ctx, "stereo_retry_kernel", stereo_retry_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        if ((st = A.tp.pass2(ctx, left, right, prm, n, nklt_pyr_lvl, A.right)) != OV2_OK) return st;
        OV2_LAUNCH(ctx, "stereo_gate_kernel", stereo_gate_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        return OV2_OK;
    });
}
