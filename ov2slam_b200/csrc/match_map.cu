// 8f-4: local-map matching - the data-parallel core of Mapper::matchToMap.
//
// Reference behaviour replaced: the body of the loop over the local map points in Mapper::matchToMap
// (/root/reference/src/mapper.cpp:601-752) and the per-keypoint selection that follows it (:754-772), on FLATTENED arrays
// (the map walking that produces them - which map points are candidates, the keyframes' observation sets and pixels, the
// keypoints' grid - is the host shim's job, as for localBA):
//   project the map point into the frame (Frame::projWorldToCam + CameraCalibration::projectCamToImageDist, pinhole or
//   pinhole + radial-tangential distortion as cv::projectPoints evaluates it on the float-rounded normalised point),
//   cull (depth < 0.1, view angle, outside the image), visit the keypoints of the FOUR grid cells
//   Frame::getSurroundingKeypoints(pt) visits (src/frame.cpp:624-650), and for each: pixel distance, "never observed
//   together" (keyframe bit sets disjoint), mean co-projection error into the keyframes observing the keypoint's map point,
//   minimal Hamming distance over all descriptor pairs (src/map_point.cpp:236-252); best / second-best with the reference's
//   `<=` update order and the 0.9 ratio test; then per keypoint the candidate with the smallest distance (later
//   candidates win ties).
// match_mp_kernel: one warp per candidate map point, a lane per surrounding keypoint (32 at a time), the order-dependent
// best / second scan replayed in keypoint order from the lanes' results.  match_kp_kernel: one thread per keypoint.
// double arithmetic without FMA contraction (-fmad=false) in OpenCV's / the reference's operation order.
#include "ov2_common.cuh"
#include "cam_project.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int WARPS = 4;

struct MatchDev {
    double Tcw[12];
    CamModel cam;
    int img_w, img_h, ncellsize, nbwcells, ncells;
    const int32_t* cell_ptr; const int32_t* cell_kp;
    int nkps; const float2* kp_px; const int32_t* kp_lm;
    int nmps; const double* mp_xyz; const int32_t* mp_desc_ptr; const uint8_t* desc; const unsigned long long* mp_kfmask;
    const int32_t* mp_obs_ptr; const int32_t* obs_kf; const float2* obs_px;
    const double* kf_Tcw;
    int ncand; const int32_t* cand_mp;
    float dmaxpxdist, mindist, view_th;
    int32_t* best_kp; float* best_dist;
    int32_t* kp_match; float* kp_dist;
};

__device__ __forceinline__ int hamming256(const uint8_t* a, const uint8_t* b) {
    const uint32_t* pa = reinterpret_cast<const uint32_t*>(a);
    const uint32_t* pb = reinterpret_cast<const uint32_t*>(b);
    int s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += __popc(pa[k] ^ pb[k]);
    return s;
}

__global__ void __launch_bounds__(WARPS * 32) match_mp_kernel(MatchDev A) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ci = blockIdx.x * WARPS + warp;
    if (ci >= A.ncand) return;
    int bestid = -1, secid = -1;
    float bestdist = A.mindist, secdist = A.mindist;
    const int mp = A.cand_mp[ci];
    const double wpt[3] = {A.mp_xyz[3 * (size_t)mp], A.mp_xyz[3 * (size_t)mp + 1], A.mp_xyz[3 * (size_t)mp + 2]};
    double X, Y, Z;
    transform(A.Tcw, wpt, X, Y, Z);
    bool alive = !(Z < 0.1);
    float2 proj = make_float2(0.f, 0.f);
    if (alive) {
        const float view_angle = (float)(Z / sqrt(X * X + Y * Y + Z * Z));
        if (fabsf(view_angle) < A.view_th) alive = false;
    }
    if (alive) {
        proj = project_dist(A.cam, X, Y, Z);
        if (!in_image(proj, A.img_w, A.img_h)) alive = false;
    }
    if (alive) {
        const int rkp = (int)floor((double)(proj.y / (float)A.ncellsize)), ckp = (int)floor((double)(proj.x / (float)A.ncellsize));
        const unsigned long long m0 = A.mp_kfmask[4 * (size_t)mp], m1 = A.mp_kfmask[4 * (size_t)mp + 1],
                                 m2 = A.mp_kfmask[4 * (size_t)mp + 2], m3 = A.mp_kfmask[4 * (size_t)mp + 3];
        const int dm0 = A.mp_desc_ptr[mp], dm1 = A.mp_desc_ptr[mp + 1];
        for (int cell4 = 0; cell4 < 4; ++cell4) {
            const int r = rkp - 1 + (cell4 >> 1), c = ckp - 1 + (cell4 & 1);
            const int idx = r * A.nbwcells + c;
            if (r < 0 || c < 0 || idx >= A.ncells) continue;
            const int q0 = A.cell_ptr[idx], q1 = A.cell_ptr[idx + 1];
            for (int base = q0; base < q1; base += 32) {
                const int q = base + lane;
                int kpid = -1;
                float d = 0.f;
                if (q < q1) {
                    const int j = A.cell_kp[q];
                    const int lm = A.kp_lm[j];
                    bool ok = lm >= 0;
                    if (ok) {
                        const float2 kp = A.kp_px[j];
                        const float dx = proj.x - kp.x, dy = proj.y - kp.y;
                        const float pxdist = (float)sqrt((double)dx * (double)dx + (double)dy * (double)dy);
                        ok = !(pxdist > A.dmaxpxdist);
                    }
                    int dl0 = 0, dl1 = 0;
                    if (ok) {
                        dl0 = A.mp_desc_ptr[lm]; dl1 = A.mp_desc_ptr[lm + 1];
                        ok = dl1 > dl0;
                    }
                    if (ok) {
                        const unsigned long long* km = A.mp_kfmask + 4 * (size_t)lm;
                        ok = ((m0 & km[0]) | (m1 & km[1]) | (m2 & km[2]) | (m3 & km[3])) == 0ull;   // never observed together
                    }
                    if (ok) {
                        float coproj = 0.f;
                        int nb = 0;
                        for (int o = A.mp_obs_ptr[lm]; o < A.mp_obs_ptr[lm + 1]; ++o) {
                            double cx_, cy_, cz_;
                            transform(A.kf_Tcw + 12 * (size_t)A.obs_kf[o], wpt, cx_, cy_, cz_);
                            const float2 pq = project_dist(A.cam, cx_, cy_, cz_);
                            const float2 op = A.obs_px[o];
                            const float ex = op.x - pq.x, ey = op.y - pq.y;
                            coproj = (float)((double)coproj + sqrt((double)ex * (double)ex + (double)ey * (double)ey));
                            nb++;
                        }
                        if (nb > 0 && coproj / (float)nb > A.dmaxpxdist) ok = false;
                    }
                    if (ok) {
                        int best = 1000;
                        for (int a = dm0; a < dm1; ++a)
                            for (int b = dl0; b < dl1; ++b) {
                                const int hd = hamming256(A.desc + 32 * (size_t)a, A.desc + 32 * (size_t)b);
                                best = hd < best ? hd : best;
                            }
                        d = (float)best;
                        kpid = j;
                    }
                }
                // the reference's order-dependent best / second update, replayed in keypoint order (mapper.cpp:726-737)
                const unsigned have = __ballot_sync(FULL, kpid >= 0);
                for (unsigned m = have; m; m &= m - 1) {
                    const int src = __ffs(m) - 1;
                    const float dd = __shfl_sync(FULL, d, src);
                    const int jj = __shfl_sync(FULL, kpid, src);
                    if (dd <= bestdist) { secdist = bestdist; secid = bestid; bestdist = dd; bestid = jj; }
                    else if (dd <= secdist) { secdist = dd; secid = jj; }
                }
            }
        }
        if (bestid != -1 && secid != -1 && 0.9 * (double)secdist < (double)bestdist) bestid = -1;
    }
    if (lane == 0) {
        A.best_kp[ci] = bestid;
        A.best_dist[ci] = bestid >= 0 ? bestdist : 0.f;
    }
}

__global__ void match_kp_kernel(MatchDev A) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= A.nkps) return;
    float bd = 1024.f;
    int bc = -1;
    for (int ci = 0; ci < A.ncand; ++ci)
        if (A.best_kp[ci] == j && A.best_dist[ci] <= bd) { bd = A.best_dist[ci]; bc = ci; }   // later candidates win ties (:764)
    A.kp_match[j] = bc;
    A.kp_dist[j] = bd;
}

}  // namespace

extern "C" ov2_status ov2_match_to_map(ov2_ctx* ctx, const ov2_match_problem* p, int32_t* best_kp_out, float* best_dist_out,
                                       int32_t* kp_match_out, float* kp_dist_out) {
    if (!ctx || !p || !best_kp_out || !best_dist_out || !kp_match_out || !kp_dist_out)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_match_to_map: bad arguments");
    if (p->ncand < 0 || p->nkps < 0 || p->nmps < 0 || p->ncellsize <= 0 || p->nbwcells <= 0 || p->ncells <= 0 || p->nkfs < 0 || p->nkfs > 256)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_match_to_map: bad sizes (at most 256 local keyframes)");
    if (p->ncand == 0 && p->nkps == 0) return OV2_OK;      // mapper.cpp:581-583: empty local map -> no match
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    MatchDev A;
    memcpy(A.Tcw, p->Tcw, sizeof(A.Tcw));
    A.cam = make_cam(p->K, p->dist);
    A.img_w = p->img_w; A.img_h = p->img_h; A.ncellsize = p->ncellsize; A.nbwcells = p->nbwcells; A.ncells = p->ncells;
    A.nkps = p->nkps; A.nmps = p->nmps; A.ncand = p->ncand;
    A.dmaxpxdist = p->dmaxpxdist; A.view_th = p->view_th;
    A.mindist = (float)((double)(32.0f * p->fdistratio) * 8.0);       // plm->desc_.cols * fdistratio * 8. (mapper.cpp:643)
    const size_t nkps = (size_t)p->nkps, nmps = (size_t)p->nmps;
    if ((st = ov2_stage_in(ctx, p->cell_ptr, (size_t)(p->ncells + 1), A.cell_ptr)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->cell_kp, nkps, A.cell_kp)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->kp_px, nkps, A.kp_px)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->kp_lm, nkps, A.kp_lm)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->mp_xyz, 3 * nmps, A.mp_xyz)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->mp_desc_ptr, nmps + 1, A.mp_desc_ptr)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->desc, 32 * (size_t)p->ndesc, A.desc)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->mp_kfmask, 4 * nmps, A.mp_kfmask)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->mp_obs_ptr, nmps + 1, A.mp_obs_ptr)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->obs_kf, (size_t)p->nobs, A.obs_kf)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->obs_px, (size_t)p->nobs, A.obs_px)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->kf_Tcw, 12 * (size_t)p->nkfs, A.kf_Tcw)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, p->cand_mp, (size_t)p->ncand, A.cand_mp)) != OV2_OK) return st;
    const size_t nout_cand = p->ncand > 0 ? p->ncand : 1, nout_kps = p->nkps > 0 ? p->nkps : 1;
    if ((st = ov2_stage_out(ctx, best_kp_out, nout_cand, A.best_kp)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, best_dist_out, nout_cand, A.best_dist)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, kp_match_out, nout_kps, A.kp_match)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, kp_dist_out, nout_kps, A.kp_dist)) != OV2_OK) return st;
    if (p->ncand > 0) OV2_LAUNCH(ctx, "match_mp_kernel", match_mp_kernel<<<div_up(p->ncand, WARPS), WARPS * 32, 0, ctx->stream>>>(A));
    if (p->nkps > 0) OV2_LAUNCH(ctx, "match_kp_kernel", match_kp_kernel<<<div_up(p->nkps, 128), 128, 0, ctx->stream>>>(A));
    return ov2_end(ctx);
}
