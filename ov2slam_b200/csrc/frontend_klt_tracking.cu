// VisualFrontEnd::kltTracking (/root/reference/src/visual_front_end.cpp:132-275) for a batch of frames, composed from the
// fbKltTracking entry point (ov2_fb_klt, frontend_klt.cu) without a host synchronisation between its steps:
//
//   klt_prior_kernel   projects every 3-D keypoint's map point into its frame (cam_project.cuh) and writes the pass-1
//                      arrays: a 3-D keypoint whose prior passes Frame::isInImage tracks from that prior, every other slot
//                      is an empty slot (x = -1), which ov2_fb_klt skips at no cost.
//   ov2_fb_klt         pass 1 over all n slots at depth 1 (:189-199).
//   klt_retry_kernel   counts the frame's pass-1 tracks (nbgood / nbkps), raises the P3P request when
//                      nbgood < 0.33 * nbkps (:228-233) and writes the pass-2 arrays: the 2-D keypoints, the 3-D keypoints
//                      without an in-image prior and the failed pass-1 keypoints; the last start from their pass-1 forward
//                      result, or from their own position when the P3P request is raised.
//   ov2_fb_klt         pass 2 over all n slots at depth nklt_pyr_lvl (:235-252); it writes the tracked positions in place.
//   klt_merge_kernel   the final status of every keypoint.
//
// All three kernels run one CTA of KT_THREADS threads per frame, each thread striding over the frame's keypoints, so a
// frame's count needs no atomics and a CTA's work is bounded by its frame's keypoint count.  The step is a fixed sequence of
// launches on the context's stream (in batch mode inside); with device arrays its only copy is the host offsets table, and
// the call returns without waiting for the stream.
#include "ov2_common.cuh"
#include "cam_project.cuh"

namespace {

constexpr int KT_THREADS = 256;

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
    // pass-1 and pass-2 slot arrays (device scratch) and the outputs
    int32_t* frame_idx;
    float2* kp1; float2* pri1; uint8_t* st1;
    float2* kp2; float2* tracked; uint8_t* st2;
    uint8_t* status; uint8_t* pass;
    uint8_t* p3p_req; int32_t* nbgood; int32_t* nbkps;
};

// Launch: grid = count, block = KT_THREADS; keypoint i of frame f is visited by thread (i - offsets[f]) % KT_THREADS.
__global__ void __launch_bounds__(KT_THREADS) klt_prior_kernel(KtArgs A) {
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    const CamModel cam = make_cam(A.K + 4 * (size_t)f, A.dist ? A.dist + 5 * (size_t)f : nullptr);
    const double* T = A.Tcw + 12 * (size_t)f;
    const int img_w = A.img_wh[2 * f], img_h = A.img_wh[2 * f + 1];
    for (int i = o0 + threadIdx.x; i < o1; i += KT_THREADS) {
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
        A.frame_idx[i] = A.first + f;
        A.kp1[i] = prior ? px : make_float2(-1.f, -1.f);
        A.pri1[i] = prior ? proj : px;
    }
}

// Launch: as klt_prior_kernel.  The frame's counts are a CTA reduction of per-thread counts (integers: order independent).
__global__ void __launch_bounds__(KT_THREADS) klt_retry_kernel(KtArgs A) {
    __shared__ int s_good[KT_THREADS / 32], s_kps[KT_THREADS / 32];
    const int f = blockIdx.x;
    const int o0 = A.offsets[f], o1 = A.offsets[f + 1];
    int good = 0, kps = 0;
    for (int i = o0 + threadIdx.x; i < o1; i += KT_THREADS) {
        const bool in1 = A.kp1[i].x >= 0.f;
        kps += in1;
        good += in1 && A.st1[i];
    }
    good = __reduce_add_sync(0xffffffffu, good);
    kps = __reduce_add_sync(0xffffffffu, kps);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_good[warp] = good; s_kps[warp] = kps; }
    __syncthreads();
    good = 0;
    kps = 0;
    for (int k = 0; k < KT_THREADS / 32; ++k) { good += s_good[k]; kps += s_kps[k]; }
    // visual_front_end.cpp:228: size_t counts against a double; no pass 1 (nbkps = 0) raises nothing
    const bool p3p = (double)good < 0.33 * (double)kps;
    if (threadIdx.x == 0) {
        A.p3p_req[f] = p3p;
        A.nbgood[f] = good;
        A.nbkps[f] = kps;
    }
    for (int i = o0 + threadIdx.x; i < o1; i += KT_THREADS) {
        const float2 px = A.px[i];
        const bool in1 = A.kp1[i].x >= 0.f;
        if (in1 && A.st1[i]) {
            // tracked with its prior: an empty slot of pass 2 that keeps the pass-1 result
            A.kp2[i] = make_float2(-1.f, -1.f);
            A.tracked[i] = A.pri1[i];
            A.pass[i] = 1;
        } else {
            A.kp2[i] = px;
            A.tracked[i] = in1 && !p3p ? A.pri1[i] : px;
            A.pass[i] = px.x >= 0.f ? 2 : 0;
        }
    }
}

// Launch: as klt_prior_kernel.
__global__ void __launch_bounds__(KT_THREADS) klt_merge_kernel(KtArgs A) {
    const int f = blockIdx.x;
    for (int i = A.offsets[f] + threadIdx.x; i < A.offsets[f + 1]; i += KT_THREADS)
        A.status[i] = A.pass[i] == 1 ? 1 : A.st2[i];
}

ov2_status enqueue(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int n, int nklt_pyr_lvl,
                   KtArgs& A, const double* Tcw, const double* K, const double* dist, const int32_t* img_wh, const float* px,
                   const double* wpt, const uint8_t* is3d, const int32_t* offsets, float* tracked_out, uint8_t* status_out,
                   uint8_t* pass_out, uint8_t* p3p_req_out, int32_t* nbgood_out, int32_t* nbkps_out) {
    const size_t nn = (size_t)n, nc = (size_t)A.count;
    ov2_status st;
    const void* d = nullptr;
    void* o = nullptr;
#define IN(ptr, bytes, field, type) do { if ((st = ov2_stage_in(ctx, ptr, bytes, &d)) != OV2_OK) return st; A.field = (const type*)d; } while (0)
#define OUT(ptr, bytes, field, type) do { if ((st = ov2_stage_out(ctx, ptr, bytes, &o)) != OV2_OK) return st; A.field = (type*)o; } while (0)
#define SCRATCH(bytes, field, type) do { if ((st = ov2_scratch(ctx, bytes, &o)) != OV2_OK) return st; A.field = (type*)o; } while (0)
    IN(offsets, sizeof(int32_t) * (nc + 1), offsets, int32_t);
    IN(Tcw, sizeof(double) * 12 * nc, Tcw, double);
    IN(K, sizeof(double) * 4 * nc, K, double);
    IN(dist, sizeof(double) * 5 * nc, dist, double);
    IN(img_wh, sizeof(int32_t) * 2 * nc, img_wh, int32_t);
    OUT(p3p_req_out, nc, p3p_req, uint8_t);
    OUT(nbgood_out, sizeof(int32_t) * nc, nbgood, int32_t);
    OUT(nbkps_out, sizeof(int32_t) * nc, nbkps, int32_t);
    if (n > 0) {
        IN(px, sizeof(float2) * nn, px, float2);
        IN(wpt, sizeof(double) * 3 * nn, wpt, double);
        IN(is3d, nn, is3d, uint8_t);
        OUT(tracked_out, sizeof(float2) * nn, tracked, float2);
        OUT(status_out, nn, status, uint8_t);
        OUT(pass_out, nn, pass, uint8_t);
        SCRATCH(sizeof(int32_t) * nn, frame_idx, int32_t);
        SCRATCH(sizeof(float2) * nn, kp1, float2);
        SCRATCH(sizeof(float2) * nn, pri1, float2);
        SCRATCH(nn, st1, uint8_t);
        SCRATCH(sizeof(float2) * nn, kp2, float2);
        SCRATCH(nn, st2, uint8_t);
    }
#undef IN
#undef OUT
#undef SCRATCH
    OV2_LAUNCH(ctx, "klt_prior_kernel", klt_prior_kernel<<<A.count, KT_THREADS, 0, ctx->stream>>>(A));
    if ((st = ov2_fb_klt(ctx, prev, cur, prm, n, A.frame_idx, 0, 0, nullptr, 1, (const float*)A.kp1, (float*)A.pri1, A.st1)) != OV2_OK)
        return st;
    OV2_LAUNCH(ctx, "klt_retry_kernel", klt_retry_kernel<<<A.count, KT_THREADS, 0, ctx->stream>>>(A));
    if ((st = ov2_fb_klt(ctx, prev, cur, prm, n, A.frame_idx, 0, 0, nullptr, nklt_pyr_lvl, (const float*)A.kp2, (float*)A.tracked,
                         A.st2)) != OV2_OK)
        return st;
    OV2_LAUNCH(ctx, "klt_merge_kernel", klt_merge_kernel<<<A.count, KT_THREADS, 0, ctx->stream>>>(A));
    return OV2_OK;
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
    if (ov2_is_device_ptr(offsets)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: offsets must be a host pointer");
    // every frame's CTA reads offsets[f] .. offsets[f + 1] of arrays sized offsets[count]
    if (offsets[0] != 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: offsets must start at 0 and be ascending");
    for (int k = 0; k < count; ++k)
        if (offsets[k + 1] < offsets[k]) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: offsets must start at 0 and be ascending");
    const int n = offsets[count];
    if (n > 0 && (!px || !wpt || !is3d || !tracked_out || !status_out || !pass_out))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: null array");
    if (first < 0 || first + count > prev->batch || first + count > cur->batch)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: more frames than pyramid slots");
    if (prm->win < 3 || prm->win > 31) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: nwinsize must be 3 .. 31");
    if (prev->nlev != cur->nlev || prev->w[0] != cur->w[0] || prev->h[0] != cur->h[0] || !prev->l0 || !cur->l0)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_klt_tracking: pyramids not built / mismatched");
    // batch mode inside (unless the caller has a batch open): the trackers' calls only enqueue, scratch survives between
    // them, and host outputs come back with one synchronisation at the end
    const bool own_batch = !ctx->batch;
    ov2_status st = own_batch ? ov2_batch_begin(ctx) : ov2_begin(ctx);
    if (st != OV2_OK) return st;
    KtArgs A = {};
    A.count = count;
    A.first = first;
    A.use_prior = use_prior ? 1 : 0;
    st = enqueue(ctx, prev, cur, prm, n, nklt_pyr_lvl, A, Tcw, K, dist, img_wh, px, wpt, is3d, offsets, tracked_out, status_out,
                 pass_out, p3p_req_out, nbgood_out, nbkps_out);
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
