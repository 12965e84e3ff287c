// FeatureExtractor on the GPU: host shim over the C ABI (include/ov2b200.h).
// Behaviour mirrored: /root/reference/src/feature_extractor.cpp:443-570 (detectGridFAST incl.
// cornerSubPix and the nfast_th_ adaptation), :288-440 (detectSingleScale incl. the dmaxquality_
// adaptation), :224-285 (describeBRIEF; non-contrib ORB branch by default, BRIEF-32 with -DOPENCV_CONTRIB), :575-584
// (setMask).  The front-end thread is the only caller (under map_mutex_, visual_front_end.cpp:42),
// so one lazily created context per process is enough.  No OpenCV on the hot path, no CPU fallback.
#include "feature_extractor.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <mutex>

#include "../../include/ov2b200.h"
#include "pyr_cache.hpp"
// The reference chooses its descriptor at compile time (CMakeLists.txt:12,35-39; feature_extractor.cpp:69-70,242-246).
// A build with -DOPENCV_CONTRIB gets BRIEF-32: the kernel is table-driven and the 256 test pairs come from
// opencv_contrib's generated_32.i through scripts/brief_table_from_contrib.py (writes include/ov2_brief32_pattern.h).
#ifdef OPENCV_CONTRIB
#include "../../include/ov2_brief32_pattern.h"
#endif

namespace {
struct State {
    ov2_ctx* ctx = nullptr;
    ov2_pyr* pyr = nullptr;                 // the image of the current call (a slot of `cache`)
    // the tracking image and the raw image of a keyframe (map_manager.cpp:286-341: detect on `im`, describe on `imraw`,
    // twice): each is uploaded once, whatever the number of calls (pyr_cache.hpp)
    ov2shim::PyrCache<3> cache;
    bool desc_configured = false;           // BRIEF-32 table loaded (contrib builds)
    std::mutex mu;
};
State& st() { static State s; return s; }

// make `im` the current device image (uploaded only if it is not already there); false (and reports) on failure
bool load_image(State& s, const cv::Mat& im) {
    if (!s.ctx) {
        // the reference's class takes no device: OV2_DEVICE names the GPU (default 0)
        const char* e = getenv("OV2_DEVICE");
        if (ov2_create(e ? atoi(e) : 0, &s.ctx) != OV2_OK) {
            fprintf(stderr, "[ov2b200] FeatureExtractor: no CUDA device - the GPU front-end has no CPU fallback\n");
            s.ctx = nullptr;
            return false;
        }
    }
#ifdef OPENCV_CONTRIB
    if (!s.desc_configured) {
        if (ov2_describe_config(s.ctx, OV2_DESC_BRIEF32, &OV2_BRIEF32_PATTERN[0][0]) != OV2_OK) {
            fprintf(stderr, "[ov2b200] FeatureExtractor: %s\n", ov2_last_error(s.ctx));
            return false;
        }
        s.desc_configured = true;
    }
#endif
    s.pyr = s.cache.get(s.ctx, im, 0);
    if (!s.pyr) {
        fprintf(stderr, "[ov2b200] FeatureExtractor: %s\n", ov2_last_error(s.ctx));
        return false;
    }
    return true;
}
}  // namespace

FeatureExtractor::FeatureExtractor(size_t nmaxpts, size_t nmaxdist, double dmaxquality, int nfast_th)
    : nmaxpts_(nmaxpts), nmaxdist_(nmaxdist), dmaxquality_(dmaxquality), nfast_th_(nfast_th)
{
    nmindist_ = nmaxdist / 2.;
    dminquality_ = dmaxquality / 2.;
}

std::vector<cv::Point2f> FeatureExtractor::detectGridFAST(const cv::Mat &im, const int ncellsize,
        const std::vector<cv::Point2f> &vcurkps, const cv::Rect &/*roi: unused by the reference too*/)
{
    if (im.empty()) return std::vector<cv::Point2f>();           // feature_extractor.cpp:446-449
    State& s = st();
    std::lock_guard<std::mutex> lk(s.mu);
    if (!load_image(s, im)) return std::vector<cv::Point2f>();
    const int ncells = (im.rows / ncellsize) * (im.cols / ncellsize);
    if (ncells <= 0) return std::vector<cv::Point2f>();
    std::vector<cv::Point2f> out((size_t)ncells);
    int32_t offsets[2] = {0, (int32_t)vcurkps.size()};
    int32_t th = nfast_th_, count = 0;
    ov2_status rc = ov2_grid_fast(s.ctx, s.pyr, 0, 1, ncellsize, vcurkps.empty() ? nullptr : offsets,
                                  vcurkps.empty() ? nullptr : reinterpret_cast<const float*>(vcurkps.data()), &th, ncells,
                                  reinterpret_cast<float*>(out.data()), &count, nullptr, 1);
    if (rc != OV2_OK) {
        fprintf(stderr, "[ov2b200] detectGridFAST: %s\n", ov2_last_error(s.ctx));
        return std::vector<cv::Point2f>();
    }
    nfast_th_ = th;                                              // adaptive threshold state (:546-552)
    out.resize((size_t)count);
    return out;
}

std::vector<cv::Mat> FeatureExtractor::describeBRIEF(const cv::Mat &im, const std::vector<cv::Point2f> &vpts) const
{
    if (vpts.empty()) return std::vector<cv::Mat>();             // :226-229
    State& s = st();
    std::lock_guard<std::mutex> lk(s.mu);
    const size_t n = vpts.size();
    std::vector<cv::Mat> vdescs(n);                              // empty cv::Mat = "not describable" (:263-278)
    if (!load_image(s, im)) return vdescs;
    cv::Mat descs((int)n, 32, CV_8U);                            // one jointly owned buffer, rows handed out
    std::vector<uint8_t> valid(n, 0);
    ov2_status rc = ov2_describe(s.ctx, s.pyr, (int)n, nullptr, 0, (int)n, reinterpret_cast<const float*>(vpts.data()),
                                 descs.data, valid.data());
    if (rc != OV2_OK) {
        fprintf(stderr, "[ov2b200] describeBRIEF: %s\n", ov2_last_error(s.ctx));
        return vdescs;
    }
    for (size_t i = 0; i < n; ++i)
        if (valid[i]) vdescs[i] = descs.row((int)i);
    return vdescs;
}

std::vector<cv::Point2f> FeatureExtractor::detectGFTT(const cv::Mat &, const std::vector<cv::Point2f> &, const cv::Mat &, int) const
{
    fprintf(stderr, "[ov2b200] detectGFTT is not built; use use_fast: 1 or use_singlescale_detector: 1 configs\n");
    return std::vector<cv::Point2f>();
}

std::vector<cv::Point2f> FeatureExtractor::detectSingleScale(const cv::Mat &im, const int ncellsize,
        const std::vector<cv::Point2f> &vcurkps, const cv::Rect &roi)
{
    if (im.empty()) return std::vector<cv::Point2f>();           // feature_extractor.cpp:290-293
    State& s = st();
    std::lock_guard<std::mutex> lk(s.mu);
    if (!load_image(s, im)) return std::vector<cv::Point2f>();
    const int ncells = (im.rows / ncellsize) * (im.cols / ncellsize);
    if (ncells <= 0) return std::vector<cv::Point2f>();
    std::vector<cv::Point2f> out((size_t)ncells);
    int32_t offsets[2] = {0, (int32_t)vcurkps.size()};
    const int32_t roi_xywh[4] = {roi.x, roi.y, roi.width, roi.height};
    double quality = dmaxquality_;
    int32_t count = 0;
    ov2_status rc = ov2_detect_single_scale(s.ctx, s.pyr, 0, 1, ncellsize, vcurkps.empty() ? nullptr : offsets,
                                            vcurkps.empty() ? nullptr : reinterpret_cast<const float*>(vcurkps.data()),
                                            roi_xywh, &quality, ncells, reinterpret_cast<float*>(out.data()), &count, nullptr, 1);
    if (rc != OV2_OK) {
        fprintf(stderr, "[ov2b200] detectSingleScale: %s\n", ov2_last_error(s.ctx));
        return std::vector<cv::Point2f>();
    }
    dmaxquality_ = quality;                                      // adaptive quality state (:418-423)
    out.resize((size_t)count);
    return out;
}

// Host utility (not on the hot path): 8-bit mask with filled discs, OpenCV's midpoint rasterisation.
void FeatureExtractor::setMask(const cv::Mat &im, const std::vector<cv::Point2f> &vpts, const int dist, cv::Mat &mask) const
{
    if (mask.empty()) {
        mask = cv::Mat(im.rows, im.cols, CV_8UC1);
        for (int r = 0; r < mask.rows; ++r) memset(mask.ptr(r), 255, (size_t)mask.cols);
    }
    std::vector<int> hw((size_t)dist + 1, -1);
    int err = 0, dx = dist, dy = 0, plus = 1, minus = (dist << 1) - 1;
    while (dx >= dy) {
        if (dx > hw[dy]) hw[dy] = dx;
        if (dy > hw[dx]) hw[dx] = dy;
        dy++; err += plus; plus += 2;
        int m = (err <= 0) - 1;
        err -= minus & m; dx += m; minus -= m & 2;
    }
    for (const auto& pt : vpts) {
        const int cx = (int)lrintf(pt.x), cy = (int)lrintf(pt.y);
        for (int d = -dist; d <= dist; ++d) {
            const int y = cy + d;
            if (y < 0 || y >= mask.rows) continue;
            const int h = hw[d < 0 ? -d : d];
            int x0 = cx - h, x1 = cx + h;
            if (x0 < 0) x0 = 0;
            if (x1 >= mask.cols) x1 = mask.cols - 1;
            if (x0 <= x1) memset(mask.ptr(y) + x0, 0, (size_t)(x1 - x0 + 1));
        }
    }
}
