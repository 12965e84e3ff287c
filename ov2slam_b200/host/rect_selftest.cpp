// Drives the CameraCalibration::rectifyImage drop-in (host/camera_calibration_rect_gpu.cpp) the way the reference does: a
// CV_16SC2 + CV_16UC1 calibration (setUndistStereoMap) called twice on a source that is a ROI of a wider buffer, a CV_32FC1
// calibration (setUndistMap), the first calibration again in place (rectifyImage(im0, im0), ov2slam.cpp:255) and a
// calibration without maps (rect = img).  Writes the four rectified images; tests/test_rect_shim.py compares them with
// cv2.remap (GPU) or with the mocked device call's rule (CPU).
//   rect_selftest in.bin out.bin      in.bin = int32 w, h | image [h][w] | map1 int16 [h][w][2] | map2 uint16 [h][w] |
//                                              map_x float [h][w] | map_y float [h][w]
#include <cstdio>
#include <cstring>
#include <vector>

#include "camera_calibration.hpp"

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int wh[2];
    if (fread(wh, 4, 2, f) != 2) return 2;
    const int w = wh[0], h = wh[1], pad = 13;
    const size_t n = (size_t)w * h;
    std::vector<unsigned char> img(n);
    CameraCalibration fixed, flt, none;
    fixed.undist_map_x_ = cv::Mat(h, w, CV_16SC2);
    fixed.undist_map_y_ = cv::Mat(h, w, CV_16UC1);
    flt.undist_map_x_ = cv::Mat(h, w, CV_32FC1);
    flt.undist_map_y_ = cv::Mat(h, w, CV_32FC1);
    bool ok = fread(img.data(), 1, n, f) == n && fread(fixed.undist_map_x_.data, 4, n, f) == n && fread(fixed.undist_map_y_.data, 2, n, f) == n &&
              fread(flt.undist_map_x_.data, 4, n, f) == n && fread(flt.undist_map_y_.data, 4, n, f) == n;
    fclose(f);
    if (!ok) return 2;
    std::vector<unsigned char> wide((size_t)(w + pad) * h, 7);
    for (int y = 0; y < h; ++y) memcpy(&wide[(size_t)y * (w + pad)], &img[(size_t)y * w], (size_t)w);
    const cv::Mat roi(h, w, CV_8UC1, wide.data(), (size_t)(w + pad));
    const cv::Mat src(h, w, CV_8UC1, img.data());

    cv::Mat r1, r2, r3;
    fixed.rectifyImage(roi, r1);
    fixed.rectifyImage(roi, r2);
    flt.rectifyImage(src, r3);
    cv::Mat inplace(h, w, CV_8UC1);
    for (int y = 0; y < h; ++y) memcpy(inplace.ptr(y), roi.ptr(y), (size_t)w);
    const unsigned char* before = inplace.data;
    fixed.rectifyImage(inplace, inplace);
    cv::Mat same;
    none.rectifyImage(src, same);
    if (r1.empty() || r2.empty() || r3.empty() || inplace.empty()) return 3;
    if (inplace.data != before) return 4;                     // in place: the image's own buffer receives the result
    if (same.data != src.data) return 5;                      // no map: rect = img (the same pixels, no copy)
    for (int y = 0; y < h; ++y)
        if (memcmp(roi.ptr(y) + w, std::vector<unsigned char>(pad, 7).data(), pad) != 0) return 6;   // the ROI's parent untouched
    FILE* g = fopen(argv[2], "wb");
    if (!g) return 7;
    for (const cv::Mat* m : {&r1, &r2, &r3, &inplace})
        for (int y = 0; y < h; ++y) fwrite(m->ptr(y), 1, (size_t)w, g);
    fclose(g);
    printf("rectifyImage drop-in: %d x %d ok\n", w, h);
    return 0;
}
