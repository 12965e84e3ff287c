/* TEST HELPER (not part of the product): an LD_PRELOAD interposer that replaces the device calls of the
 * CameraCalibration::rectifyImage drop-in (ov2slam_b200/host/camera_calibration_rect_gpu.cpp) by a RECORDER with a rule-based
 * answer, so its host-side flow (map cache, strides, in-place calls, the no-map copy) can be checked on a box without a GPU.
 * Every call is appended to $OV2_MOCK_LOG as 10 int32:
 *   ov2_remap_create  6, map_type, width, height, map1_stride, map2_stride, 0, 0, 0, 0
 *   ov2_remap         5, map_type, width, height, src_row_stride, src_frame_stride, dst_row_stride, dst_frame_stride, count, src == dst
 *   remap rule        dst = 255 - src (row strides honoured; host buffers, the source read before the destination is written) */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/ov2b200.h"

static int dummy_ctx;
struct ov2_remap_map { int type, w, h; };

static void log_rec(const int32_t rec[10]) {
    const char* path = getenv("OV2_MOCK_LOG");
    FILE* f = path ? fopen(path, "ab") : NULL;
    if (f) { fwrite(rec, 4, 10, f); fclose(f); }
}

ov2_status ov2_create(int device, ov2_ctx** out) { (void)device; *out = (ov2_ctx*)&dummy_ctx; return OV2_OK; }
void ov2_destroy(ov2_ctx* ctx) { (void)ctx; }
const char* ov2_last_error(const ov2_ctx* ctx) { (void)ctx; return "mock"; }

ov2_status ov2_remap_create(ov2_ctx* ctx, int map_type, int width, int height, const void* map1, size_t map1_stride, const void* map2,
                            size_t map2_stride, ov2_remap_map** out) {
    (void)ctx; (void)map1; (void)map2;
    const int32_t rec[10] = {6, map_type, width, height, (int32_t)map1_stride, (int32_t)map2_stride, 0, 0, 0, 0};
    log_rec(rec);
    ov2_remap_map* m = (ov2_remap_map*)malloc(sizeof(ov2_remap_map));
    m->type = map_type; m->w = width; m->h = height;
    *out = m;
    return OV2_OK;
}

void ov2_remap_destroy(ov2_remap_map* map) { free(map); }

ov2_status ov2_remap(ov2_ctx* ctx, const ov2_remap_map* map, const uint8_t* src, size_t src_row_stride, size_t src_frame_stride,
                     uint8_t* dst, size_t dst_row_stride, size_t dst_frame_stride, int count) {
    (void)ctx;
    const int32_t rec[10] = {5, map->type, map->w, map->h, (int32_t)src_row_stride, (int32_t)src_frame_stride, (int32_t)dst_row_stride,
                             (int32_t)dst_frame_stride, count, src == dst};
    log_rec(rec);
    uint8_t* tmp = (uint8_t*)malloc((size_t)map->w * map->h);
    for (int y = 0; y < map->h; ++y) memcpy(tmp + (size_t)y * map->w, src + (size_t)y * src_row_stride, (size_t)map->w);
    for (int y = 0; y < map->h; ++y)
        for (int x = 0; x < map->w; ++x) dst[(size_t)y * dst_row_stride + x] = (uint8_t)(255 - tmp[(size_t)y * map->w + x]);
    free(tmp);
    return OV2_OK;
}
