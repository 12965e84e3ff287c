// Drop-in replacement of the reference's include/feature_tracker.hpp (:33-56): same class, same
// public members and signatures, so visual_front_end.cpp / map_manager.cpp / mapper.cpp compile
// and link against it unchanged.  fbKltTracking and inBorder run through the C ABI
// (include/ov2b200.h); getLineMinSAD (only used when bdo_stereo_rect = 1) is a statement-by-statement host port of
// the reference's function, OpenCV's 8-bit getRectSubPix template included.
#pragma once

#include <opencv2/core.hpp>
#include <opencv2/imgproc.hpp>

#include <vector>

struct ov2_ctx;
struct ov2_pyr;

class FeatureTracker {
public:
    FeatureTracker(int nmax_iter, float fmax_px_precision, cv::Ptr<cv::CLAHE> pclahe);
    ~FeatureTracker();
    FeatureTracker(const FeatureTracker&) = delete;
    FeatureTracker& operator=(const FeatureTracker&) = delete;

    // Forward-Backward KLT Tracking
    void fbKltTracking(const std::vector<cv::Mat> &vprevpyr, const std::vector<cv::Mat> &vcurpyr, int nwinsize, int nbpyrlvl, float ferr, float fmax_fbklt_dist,
        std::vector<cv::Point2f> &vpts, std::vector<cv::Point2f> &vpriorkps, std::vector<bool> &vkpstatus) const;

    void getLineMinSAD(const cv::Mat &iml, const cv::Mat &imr, const cv::Point2f &pt, const int nwinsize, float &xprior, float &l1err, bool bgoleft) const;

    bool inBorder(const cv::Point2f &pt, const cv::Mat &im) const;

    // KLT optim. parameter
    cv::TermCriteria klt_convg_crit_;

    cv::Ptr<cv::CLAHE> pclahe_;

    // fbKltTracking is const and is called concurrently from the front-end and the mapper threads
    // (map_manager.cpp:510,550): every calling thread gets its own context + pyramid slots.
    struct ThreadState;   // implementation detail
private:
    ThreadState* state() const;
};
