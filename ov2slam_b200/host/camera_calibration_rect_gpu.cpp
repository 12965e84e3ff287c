// CameraCalibration::rectifyImage on the GPU (row R of the scope table): the reference's declaration
// (/root/reference/include/camera_calibration.hpp:67) is kept, this translation unit supplies the body that
// src/camera_calibration.cpp:233-241 has (cv::remap(img, rect, undist_map_x_, undist_map_y_, cv::INTER_LINEAR), or rect = img
// when no map was built) - compiled with OV2_EXTERNAL_RECTIFY, which removes the reference's body (INTEGRATION.md section 2).
// The call goes to ov2_remap (csrc/frontend_remap.cu: bit-exact with cv::remap, tests/test_remap_gpu.py).
//
// One device context per calling thread (SlamManager::addNewStereoImages / addNewMonoImage call it from the thread that feeds
// images, src/ov2slam.cpp:239-257).  Each thread keeps its device maps in a small cache keyed on the maps' data pointers, size
// and type: the reference builds undist_map_x_ / undist_map_y_ once, in setUndistStereoMap / setUndistMap at set-up
// (camera_calibration.cpp:92,141), and never writes them afterwards, so a map seen once is converted once.  A calibration
// that rebuilt its maps in the same buffers would keep rectifying with the old ones.
// No CPU fallback: without a device, or on a CUDA error, rect is left EMPTY and the error is printed.
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "camera_calibration.hpp"       // the reference's, unchanged
#include "../../include/ov2b200.h"

namespace {

constexpr int kCV_8UC1 = 0, kCV_16UC1 = 2, kCV_32FC1 = 5, kCV_16SC2 = 11;   // OpenCV type codes (the reference's "m1type = 11")

struct MapKey {
    const void* x; const void* y; int rows, cols, type;
    bool operator==(const MapKey& o) const { return x == o.x && y == o.y && rows == o.rows && cols == o.cols && type == o.type; }
};

struct ThreadCtx {
    ov2_ctx* ctx = nullptr;
    bool tried = false;
    std::vector<std::pair<MapKey, ov2_remap_map*>> maps;
    ~ThreadCtx() {
        for (auto& m : maps) ov2_remap_destroy(m.second);
        if (ctx) ov2_destroy(ctx);
    }
};

ThreadCtx& thread_state() {
    static thread_local ThreadCtx t;
    if (!t.tried) {
        t.tried = true;
        const char* e = getenv("OV2_DEVICE");
        if (ov2_create(e ? atoi(e) : 0, &t.ctx) != OV2_OK) {
            fprintf(stderr, "[ov2b200] rectifyImage: no CUDA device - the GPU front-end has no CPU fallback\n");
            t.ctx = nullptr;
        }
    }
    return t;
}

// the device map of (map_x, map_y), created on first use
ov2_remap_map* device_map(ThreadCtx& t, const cv::Mat& mx, const cv::Mat& my) {
    const MapKey key{mx.data, my.data, mx.rows, mx.cols, mx.type()};
    for (auto& m : t.maps)
        if (m.first == key) return m.second;
    int type = 0;
    if (mx.type() == kCV_16SC2 && my.type() == kCV_16UC1) type = OV2_MAP_16SC2;
    else if (mx.type() == kCV_32FC1 && my.type() == kCV_32FC1) type = OV2_MAP_32FC1;
    else {
        fprintf(stderr, "[ov2b200] rectifyImage: maps must be CV_16SC2 + CV_16UC1 or CV_32FC1 x 2\n");
        return nullptr;
    }
    if (my.rows != mx.rows || my.cols != mx.cols) {
        fprintf(stderr, "[ov2b200] rectifyImage: the two maps differ in size\n");
        return nullptr;
    }
    ov2_remap_map* m = nullptr;
    if (ov2_remap_create(t.ctx, type, mx.cols, mx.rows, mx.data, mx.step, my.data, my.step, &m) != OV2_OK) {
        fprintf(stderr, "[ov2b200] rectifyImage: %s\n", ov2_last_error(t.ctx));
        return nullptr;
    }
    t.maps.emplace_back(key, m);
    return m;
}

}  // namespace

void CameraCalibration::rectifyImage(const cv::Mat &img, cv::Mat &rect) const
{
    std::lock_guard<std::mutex> lock(intrinsic_mutex_);

    if (undist_map_x_.empty()) {
        rect = img;
        return;
    }
    ThreadCtx& t = thread_state();
    ov2_remap_map* m = t.ctx ? device_map(t, undist_map_x_, undist_map_y_) : nullptr;
    if (!m || img.type() != kCV_8UC1 || img.rows != undist_map_x_.rows || img.cols != undist_map_x_.cols) {
        if (m) fprintf(stderr, "[ov2b200] rectifyImage: 8-bit one-channel images of the map's size only\n");
        rect = cv::Mat();
        return;
    }
    rect.create(img.rows, img.cols, kCV_8UC1);      // a no-op when rect is img (in place, as the reference calls it)
    // host buffers: ov2_remap uploads the source before it writes the destination, so rect may share img's pixels
    if (ov2_remap(t.ctx, m, img.data, img.step, 0, rect.data, rect.step, 0, 1) != OV2_OK) {
        fprintf(stderr, "[ov2b200] rectifyImage: %s\n", ov2_last_error(t.ctx));
        rect = cv::Mat();
    }
}
