// Minimal STAND-IN for the reference's include/visual_front_end.hpp: the members VisualFrontEnd::kltTracking reads and writes
// (visual_front_end.hpp:129-141), with the reference's names, for compile-checking and self-testing
// ov2slam_b200/host/visual_front_end_klt_gpu.cpp without the reference's dependencies.  On a box that builds the reference, its
// own header is used instead.
#pragma once
#include <memory>
#include <vector>

#include <opencv2/core.hpp>

#include "map_manager.hpp"

class VisualFrontEnd {
public:
    void kltTracking();

    std::shared_ptr<SlamParams> pslamstate_;
    std::shared_ptr<Frame> pcurframe_;
    std::shared_ptr<MapManager> pmap_;
    std::shared_ptr<FeatureTracker> ptracker_;
    std::vector<cv::Mat> cur_pyr_, prev_pyr_;
    bool bp3preq_ = false;
};
