/* Replaces the device calls the drop-in VisualFrontEnd::kltTracking makes (context, pyramid slots, ov2_klt_tracking) by a
 * RECORDER with canned, rule-based answers, so its host-side flow (flattening, side effects) runs on a machine without a GPU.
 * Loaded with LD_PRELOAD by tests/test_klt_tracking_shim.py.
 *
 * Log (OV2_MOCK_LOG): per ov2_pyr_build "B"; per ov2_klt_tracking "K", then i32 first, count, n, win, max_iter, nklt_pyr_lvl,
 * use_prior, has_dist, img_wh[2]; f32 eps, ferr, fb_dist; f64 Tcw[12], K[4], dist[5] (zeros without); per keypoint f32 px[2],
 * f64 wpt[3], u8 is3d.
 * Answers for keypoint i: a 3-D keypoint with i % 2 == 0 is a pass-1 track (pass 1, status 1, tracked = px + (1, 2)); every other
 * keypoint is a pass-2 keypoint (pass 2, tracked = px + (3, 4)), status 0 when i % 3 == 0; p3p_req = use_prior. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/ov2b200.h"

static int dummy_ctx;

static FILE* log_file(void) {
    static FILE* f = NULL;
    if (!f) f = fopen(getenv("OV2_MOCK_LOG"), "wb");
    return f;
}

ov2_status ov2_create(int device, ov2_ctx** out) { (void)device; *out = (ov2_ctx*)&dummy_ctx; return OV2_OK; }
void ov2_destroy(ov2_ctx* ctx) { (void)ctx; }
const char* ov2_last_error(const ov2_ctx* ctx) { (void)ctx; return "mock"; }
ov2_status ov2_pyr_create(ov2_ctx* ctx, int batch, int width, int height, int nlevels_extra, ov2_pyr** out) {
    (void)ctx; (void)batch; (void)width; (void)height; (void)nlevels_extra;
    *out = (ov2_pyr*)malloc(16);
    return OV2_OK;
}
void ov2_pyr_destroy(ov2_pyr* pyr) { free(pyr); }
ov2_status ov2_pyr_build(ov2_ctx* ctx, ov2_pyr* pyr, const uint8_t* images, size_t row_stride, size_t frame_stride, int first, int count) {
    (void)ctx; (void)pyr; (void)images; (void)row_stride; (void)frame_stride; (void)first; (void)count;
    fwrite("B", 1, 1, log_file());
    return OV2_OK;
}

ov2_status ov2_klt_tracking(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int first, int count,
                            const int32_t* offsets, const double* Tcw, const double* K, const double* dist, const int32_t* img_wh,
                            const float* px, const double* wpt, const uint8_t* is3d, int nklt_pyr_lvl, int use_prior,
                            float* tracked_out, uint8_t* status_out, uint8_t* pass_out, uint8_t* p3p_req_out, int32_t* nbgood_out,
                            int32_t* nbkps_out) {
    (void)ctx; (void)prev; (void)cur;
    FILE* f = log_file();
    const int n = offsets[count];
    const int32_t hd[10] = {first, count, n, prm->win, prm->max_iter, nklt_pyr_lvl, use_prior, dist ? 1 : 0, img_wh[0], img_wh[1]};
    const float pf[3] = {prm->eps, prm->ferr, prm->fb_dist};
    const double zero[5] = {0, 0, 0, 0, 0};
    fwrite("K", 1, 1, f);
    fwrite(hd, 4, 10, f);
    fwrite(pf, 4, 3, f);
    fwrite(Tcw, 8, 12, f);
    fwrite(K, 8, 4, f);
    fwrite(dist ? dist : zero, 8, 5, f);
    int good = 0, kps = 0;
    for (int i = 0; i < n; ++i) {
        fwrite(px + 2 * i, 4, 2, f);
        fwrite(wpt + 3 * i, 8, 3, f);
        fwrite(is3d + i, 1, 1, f);
        const int p1 = is3d[i] && i % 2 == 0;
        pass_out[i] = p1 ? 1 : 2;
        status_out[i] = p1 || i % 3 != 0;
        tracked_out[2 * i] = px[2 * i] + (p1 ? 1.f : 3.f);
        tracked_out[2 * i + 1] = px[2 * i + 1] + (p1 ? 2.f : 4.f);
        kps += is3d[i];
        good += p1;
    }
    p3p_req_out[0] = use_prior ? 1 : 0;
    nbgood_out[0] = good;
    nbkps_out[0] = kps;
    fflush(f);
    return OV2_OK;
}
