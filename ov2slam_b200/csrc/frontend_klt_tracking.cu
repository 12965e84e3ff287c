// VisualFrontEnd::kltTracking (/root/reference/src/visual_front_end.cpp:132-275) for a batch of frames, composed from the
// fbKltTracking entry point (ov2_fb_klt, frontend_klt.cu) without a host synchronisation between its steps:
//
//   klt_prior_kernel   projects every 3-D keypoint's map point into its frame (cam_project.cuh); a 3-D keypoint whose prior
//                      passes Frame::isInImage is guided, and writes the pass-1 slots.
//   ov2_fb_klt         pass 1 at depth 1 (:189-199).
//   klt_retry_kernel   counts the frame's pass-1 tracks (nbgood / nbkps), raises the P3P request when
//                      nbgood < 0.33 * nbkps (:228-233) and writes the pass-2 slots.  Every keypoint with x >= 0 is a member;
//                      a failed pass-1 keypoint restarts from its forward result, or from its own position when the P3P
//                      request is raised.
//   ov2_fb_klt         pass 2 at depth nklt_pyr_lvl (:235-252); it writes the tracked positions in place.
//   klt_merge_kernel   the final status of every keypoint.
//
// All three kernels run one CTA per frame and write the slots by the shared two-pass protocol (two_pass.cuh).  The step is a
// fixed sequence of launches on the context's stream (in batch mode inside); with device arrays its only copy is the host
// offsets table, and the call returns without waiting for the stream.
#include "ov2_common.cuh"
#include "cam_project.cuh"
#include "two_pass.cuh"

namespace {

using namespace two_pass;

struct KtArgs {
    int count, first;
    const int32_t* offsets;   // [count + 1]
    const double* Tcw;        // [count][12]
    const double* K;          // [count][4]
    const double* dist;       // [count][5] or null
    const int32_t* img_wh;    // [count][2]
    const float2* px;         // [n]
    const double* wpt;        // [n][3]
    const uint8_t* is3d;      // [n]
    int use_prior;
    TwoPass tp;
    float2* tracked; uint8_t* status; uint8_t* pass;
    uint8_t* p3p_req; int32_t* nbgood; int32_t* nbkps;
};

// Launch: grid = count, block = THREADS; keypoint i of frame f is visited by thread (i - offsets[f]) % THREADS.
__global__ void __launch_bounds__(THREADS) klt_prior_kernel(KtArgs A) {
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    const double* T = A.Tcw + 12 * (size_t)f;
    const int img_w = A.img_wh[2 * f], img_h = A.img_wh[2 * f + 1];
    for (int i = o0 + threadIdx.x; i < o1; i += THREADS) {
        const float2 px = A.px[i];
        bool prior = false;
        float2 proj = px;
        if (A.use_prior && A.is3d[i]) {
            const double w[3] = {A.wpt[3 * (size_t)i], A.wpt[3 * (size_t)i + 1], A.wpt[3 * (size_t)i + 2]};
            double X, Y, Z;
            transform(T, w, X, Y, Z);
            proj = project_dist(cam, X, Y, Z);
            prior = in_image(proj, img_w, img_h);
        }
        A.tp.set_pass1(i, A.first + f, px, prior, proj);
    }
}

// Launch: as klt_prior_kernel.
__global__ void __launch_bounds__(THREADS) klt_retry_kernel(KtArgs A) {
    __shared__ int s_good[THREADS / 32], s_kps[THREADS / 32];
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    int good = 0, kps = 0;
    for (int i = o0 + threadIdx.x; i < o1; i += THREADS) {
        const bool in1 = A.tp.kp1[i].x >= 0.f;
        kps += in1;
        good += in1 && A.tp.st1[i];
    }
    good = cta_sum(good, s_good);
    kps = cta_sum(kps, s_kps);
    // visual_front_end.cpp:228: size_t counts against a double; no pass 1 (nbkps = 0) raises nothing
    const bool p3p = (double)good < 0.33 * (double)kps;
    if (threadIdx.x == 0) {
        A.p3p_req[f] = p3p;
        A.nbgood[f] = good;
        A.nbkps[f] = kps;
    }
    for (int i = o0 + threadIdx.x; i < o1; i += THREADS) {
        const float2 px = A.px[i];
        const float2 restart = A.tp.kp1[i].x >= 0.f && !p3p ? A.tp.pri1[i] : px;
        A.tp.set_pass2(i, px, px.x >= 0.f, restart, A.tracked, A.pass);
    }
}

// Launch: as klt_prior_kernel.
__global__ void __launch_bounds__(THREADS) klt_merge_kernel(KtArgs A) {
    const int f = blockIdx.x;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += THREADS)
        A.status[i] = A.pass[i] == 1 ? 1 : A.tp.st2[i];
}

}  // namespace

extern "C" ov2_status ov2_klt_tracking(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int first,
                                       int count, const int32_t* offsets, const double* Tcw, const double* K, const double* dist,
                                       const int32_t* img_wh, const float* px, const double* wpt, const uint8_t* is3d,
                                       int nklt_pyr_lvl, int use_prior, float* tracked_out, uint8_t* status_out, uint8_t* pass_out,
                                       uint8_t* p3p_req_out, int32_t* nbgood_out, int32_t* nbkps_out) {
    if (!ctx || !prev || !cur || !prm || count < 0 || nklt_pyr_lvl < 0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: bad arguments");
    if (count == 0) return OV2_OK;
    if (!offsets || !Tcw || !K || !img_wh || !p3p_req_out || !nbgood_out || !nbkps_out)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: null array");
    const ov2_offsets_check oc = ov2_check_offsets(offsets, count);
    if (oc == OV2_OFFSETS_ON_DEVICE) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: offsets must be a host pointer");
    if (oc != OV2_OFFSETS_OK) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: offsets must start at 0 and be ascending");
    const int n = offsets[count];
    if (n > 0 && (!px || !wpt || !is3d || !tracked_out || !status_out || !pass_out))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: null array");
    if (first < 0 || first + count > prev->batch || first + count > cur->batch)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: more frames than pyramid slots");
    if (prm->win < 3 || prm->win > 31) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: nwinsize must be 3 .. 31");
    if (!ov2_pyr_pair_ok(prev, cur)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: pyramids not built / mismatched");
    return ov2_in_batch(ctx, [&]() -> ov2_status {
        const size_t nn = (size_t)n, nc = (size_t)count;
        KtArgs A = {};
        A.count = count;
        A.first = first;
        A.use_prior = use_prior ? 1 : 0;
        ov2_status st;
        if ((st = ov2_stage_in(ctx, offsets, nc + 1, A.offsets)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, Tcw, 12 * nc, A.Tcw)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, K, 4 * nc, A.K)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, dist, 5 * nc, A.dist)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, img_wh, 2 * nc, A.img_wh)) != OV2_OK) return st;
        if ((st = ov2_stage_out(ctx, p3p_req_out, nc, A.p3p_req)) != OV2_OK) return st;
        if ((st = ov2_stage_out(ctx, nbgood_out, nc, A.nbgood)) != OV2_OK) return st;
        if ((st = ov2_stage_out(ctx, nbkps_out, nc, A.nbkps)) != OV2_OK) return st;
        if (n > 0) {
            if ((st = ov2_stage_in(ctx, px, nn, A.px)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, wpt, 3 * nn, A.wpt)) != OV2_OK) return st;
            if ((st = ov2_stage_in(ctx, is3d, nn, A.is3d)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, tracked_out, nn, A.tracked)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, status_out, nn, A.status)) != OV2_OK) return st;
            if ((st = ov2_stage_out(ctx, pass_out, nn, A.pass)) != OV2_OK) return st;
            if ((st = A.tp.stage(ctx, nn)) != OV2_OK) return st;
        }
        OV2_LAUNCH(ctx, "klt_prior_kernel", klt_prior_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        if ((st = A.tp.pass1(ctx, prev, cur, prm, n)) != OV2_OK) return st;
        OV2_LAUNCH(ctx, "klt_retry_kernel", klt_retry_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        if ((st = A.tp.pass2(ctx, prev, cur, prm, n, nklt_pyr_lvl, A.tracked)) != OV2_OK) return st;
        OV2_LAUNCH(ctx, "klt_merge_kernel", klt_merge_kernel<<<count, THREADS, 0, ctx->stream>>>(A));
        return OV2_OK;
    });
}
