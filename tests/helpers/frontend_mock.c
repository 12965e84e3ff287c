/* TEST HELPER (not part of the product): an LD_PRELOAD interposer that replaces the device calls of the MapManager::stereoMatching
 * drop-in (ov2slam_b200/host/map_manager_stereo_gpu.cpp: context, pyramid slots, ov2_stereo_matching) and of the cv::CLAHE adapter
 * (ov2_clahe) by a RECORDER with canned, rule-based answers, so their host side (what they hand to the device, what they do with the
 * answers) can be checked on a box without a GPU.  Every call is appended to $OV2_MOCK_LOG (int32 tag first); tests/test_host_shim.py
 * reads the log and applies the same rules.
 *   pyramid      tag 3
 *   CLAHE        tag 4, arguments; dst = 255 - src (row strides honoured)
 *   stereo       tag 5; i32 first, count, n, win, max_iter, rectified, nklt_pyr_lvl, has_dist, has_grid, img_wh[2], ncells;
 *                f32 eps, ferr, fb_dist; f64 Tcw[12], K[4], dist[5] (zeros without), Trl[12], Frl[9]; i32 grid[2] (zeros without),
 *                with the grid i32 cell_ptr[ncells + 1], cell_kps[n]; f32 px[n][2], unpx[n][2]; f64 bv[n][3]; u8 is3d[n],
 *                has_mp[n]; f64 wpt[n][3].
 *                Answers for keypoint i: an empty slot (px.x < 0) or a 3-D keypoint without a map point is not tracked (pass 0,
 *                right = px); every other keypoint is tracked in pass 1 + i % 2 to right = px + (-10 - i % 7, 0.25), and is a
 *                stereo match iff i % 3 != 0. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/ov2b200.h"

static int dummy_ctx;
struct mock_pyr { int w, h, nlev; };

static FILE* log_file(void) {
    const char* path = getenv("OV2_MOCK_LOG");
    return path ? fopen(path, "ab") : NULL;
}

ov2_status ov2_create(int device, ov2_ctx** out) { (void)device; *out = (ov2_ctx*)&dummy_ctx; return OV2_OK; }
void ov2_destroy(ov2_ctx* ctx) { (void)ctx; }
const char* ov2_last_error(const ov2_ctx* ctx) { (void)ctx; return "mock"; }
ov2_status ov2_pyr_create(ov2_ctx* ctx, int batch, int width, int height, int nlevels_extra, ov2_pyr** out) {
    (void)ctx; (void)batch;
    struct mock_pyr* p = (struct mock_pyr*)malloc(sizeof(struct mock_pyr));
    p->w = width; p->h = height; p->nlev = nlevels_extra;
    *out = (ov2_pyr*)p;
    return OV2_OK;
}
void ov2_pyr_destroy(ov2_pyr* pyr) { free(pyr); }
ov2_status ov2_pyr_build(ov2_ctx* ctx, ov2_pyr* pyr, const uint8_t* images, size_t row_stride, size_t frame_stride, int first, int count) {
    (void)ctx; (void)pyr; (void)images; (void)row_stride; (void)frame_stride; (void)first; (void)count;
    FILE* f = log_file();
    if (f) { int32_t tag = 3; fwrite(&tag, 4, 1, f); fclose(f); }
    return OV2_OK;
}

ov2_status ov2_stereo_matching(ov2_ctx* ctx, const ov2_pyr* left, const ov2_pyr* right, const ov2_klt_params* prm, int first, int count,
                               const int32_t* offsets, const double* Tcw, const double* K, const double* dist, const double* Trl,
                               const double* Frl, const int32_t* img_wh, const int32_t* cell_offsets, const int32_t* grid,
                               const int32_t* cell_ptr, const int32_t* cell_kps, const float* px, const float* unpx, const double* bv,
                               const uint8_t* is3d, const uint8_t* has_mp, const double* wpt, int rectified, int nklt_pyr_lvl,
                               float* right_out, uint8_t* stereo_out, uint8_t* pass_out, int32_t* nstereo_out) {
    (void)ctx; (void)left; (void)right;
    const int n = offsets[count];
    const int ncells = cell_offsets ? cell_offsets[count] : 0;
    FILE* f = log_file();
    if (f) {
        const int32_t hd[13] = {5, first, count, n, prm->win, prm->max_iter, rectified, nklt_pyr_lvl, dist != NULL, cell_offsets != NULL,
                                img_wh[0], img_wh[1], ncells};
        const float pf[3] = {prm->eps, prm->ferr, prm->fb_dist};
        const double zero[5] = {0, 0, 0, 0, 0};
        const int32_t nogrid[2] = {0, 0};
        fwrite(hd, 4, 13, f); fwrite(pf, 4, 3, f);
        fwrite(Tcw, 8, 12, f); fwrite(K, 8, 4, f); fwrite(dist ? dist : zero, 8, 5, f); fwrite(Trl, 8, 12, f); fwrite(Frl, 8, 9, f);
        fwrite(grid ? grid : nogrid, 4, 2, f);
        if (cell_offsets) { fwrite(cell_ptr, 4, (size_t)ncells + 1, f); fwrite(cell_kps, 4, (size_t)n, f); }
        fwrite(px, 4, 2 * (size_t)n, f); fwrite(unpx, 4, 2 * (size_t)n, f); fwrite(bv, 8, 3 * (size_t)n, f);
        fwrite(is3d, 1, (size_t)n, f); fwrite(has_mp, 1, (size_t)n, f); fwrite(wpt, 8, 3 * (size_t)n, f);
        fclose(f);
    }
    for (int k = 0; k < count; ++k) nstereo_out[k] = 0;
    for (int k = 0; k < count; ++k)
        for (int i = offsets[k]; i < offsets[k + 1]; ++i) {
            const int tracked = px[2 * i] >= 0.f && !(is3d[i] && !has_mp[i]);
            pass_out[i] = tracked ? (uint8_t)(1 + i % 2) : 0;
            stereo_out[i] = tracked && i % 3 != 0;
            right_out[2 * i] = px[2 * i] + (tracked ? -10.f - (float)(i % 7) : 0.f);
            right_out[2 * i + 1] = px[2 * i + 1] + (tracked ? 0.25f : 0.f);
            nstereo_out[k] += stereo_out[i];
        }
    return OV2_OK;
}

ov2_status ov2_clahe(ov2_ctx* ctx, const uint8_t* src, uint8_t* dst, int width, int height, size_t row_stride, size_t frame_stride, int count,
                     double clip_limit, int tiles_x, int tiles_y) {
    (void)ctx; (void)frame_stride;
    FILE* f = log_file();
    if (f) {
        int32_t hd[8] = {4, width, height, (int32_t)row_stride, count, (int32_t)(clip_limit * 1000), tiles_x, tiles_y};
        hd[0] = 4;
        fwrite(hd, 4, 8, f);
        int32_t inplace = src == dst;
        fwrite(&inplace, 4, 1, f);
        fclose(f);
    }
    for (int y = 0; y < height; ++y)
        for (int x = 0; x < width; ++x) dst[(size_t)y * row_stride + x] = (uint8_t)(255 - src[(size_t)y * row_stride + x]);
    return OV2_OK;
}
