// cv::CLAHE over ov2_clahe (see clahe_gpu.hpp).  One device context per calling thread (apply is called from the front-end and the
// mapper threads); no CPU fallback: without a device, or on a CUDA error, the output is left EMPTY and the error is printed.
#include "clahe_gpu.hpp"

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/ov2b200.h"

namespace {

struct ThreadCtx {
    ov2_ctx* ctx = nullptr;
    bool tried = false;
    ~ThreadCtx() { if (ctx) ov2_destroy(ctx); }
};

ov2_ctx* thread_context() {
    static thread_local ThreadCtx t;
    if (!t.tried) {
        t.tried = true;
        // the reference's call takes no device: OV2_DEVICE names the GPU (default 0)
        const char* e = getenv("OV2_DEVICE");
        if (ov2_create(e ? atoi(e) : 0, &t.ctx) != OV2_OK) {
            fprintf(stderr, "[ov2b200] CLAHE: no CUDA device - the GPU front-end has no CPU fallback\n");
            t.ctx = nullptr;
        }
    }
    return t.ctx;
}

class GpuCLAHE : public cv::CLAHE {
public:
    GpuCLAHE(double clip, cv::Size tiles) : clip_(clip), tiles_(tiles) {}

#ifdef OV2_STANDIN_OPENCV
    void apply(const cv::Mat& src, cv::Mat& dst) override { run(src, dst); }
#else
    void apply(cv::InputArray _src, cv::OutputArray _dst) override {
        cv::Mat src = _src.getMat();
        CV_Assert(src.type() == CV_8UC1);                 // the reference feeds 8-bit grey images only
        _dst.create(src.size(), src.type());              // a no-op when dst IS src (in place)
        cv::Mat dst = _dst.getMat();
        run(src, dst);
        if (dst.empty()) _dst.release();
    }
    void setClipLimit(double clipLimit) override { clip_ = clipLimit; }
    double getClipLimit() const override { return clip_; }
    void setTilesGridSize(cv::Size tileGridSize) override { tiles_ = tileGridSize; }
    cv::Size getTilesGridSize() const override { return tiles_; }
    void collectGarbage() override {}
#endif

private:
    void run(const cv::Mat& src, cv::Mat& dst) {
        if (src.empty()) { dst = cv::Mat(); return; }
        if (dst.empty() || dst.rows != src.rows || dst.cols != src.cols) dst = cv::Mat(src.rows, src.cols, CV_8UC1);
        ov2_ctx* ctx = thread_context();
        if (!ctx) { dst = cv::Mat(); return; }
        const uint8_t* in = src.data;
        if (src.data != dst.data && src.step != dst.step) {
            // the ABI takes one row stride for both images: bring the source into the destination's layout and equalise in place
            // (allowed for host buffers)
            for (int r = 0; r < src.rows; ++r) memcpy(dst.ptr(r), src.ptr(r), (size_t)src.cols);
            in = dst.data;
        }
        const ov2_status st = ov2_clahe(ctx, in, dst.data, src.cols, src.rows, dst.step, 0, 1, clip_, tiles_.width, tiles_.height);
        if (st != OV2_OK) {
            fprintf(stderr, "[ov2b200] CLAHE: %s\n", ov2_last_error(ctx));
            dst = cv::Mat();
        }
    }
    double clip_;
    cv::Size tiles_;
};

}  // namespace

namespace ov2shim {
cv::Ptr<cv::CLAHE> createCLAHE(double clipLimit, cv::Size tileGridSize) { return cv::Ptr<cv::CLAHE>(new GpuCLAHE(clipLimit, tileGridSize)); }
}
