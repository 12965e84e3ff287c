// VisualFrontEnd::kltTracking on the GPU: the reference's declaration (include/visual_front_end.hpp:109) is kept, this translation
// unit supplies the body.  Exclude the reference's own body (src/visual_front_end.cpp:132-275) with #ifndef OV2_EXTERNAL_KLTTRACKING.
//
// It flattens the current frame's keypoints (mapkps_, in the map's iteration order) with their map points, the frame's pose and the
// left calibration, reads the two pyramids from the device-pyramid cache (pyr_cache.hpp) and makes ONE ov2_klt_tracking call: the
// prior projection, the depth-1 pass, the 33 % rule and the full-depth retry run on the device without a synchronisation between
// them (the reference's two fbKltTracking calls each wait for their results).  Then it applies the reference's side effects in the
// reference's order: updateKeypoint for the pass-1 tracks, bp3preq_ = true when the frame asks for P3P (never cleared here), then
// updateKeypoint or removeObsFromCurFrameById for every pass-2 keypoint.  Each side effect touches one keypoint id, so the order of
// the pass-2 list (the reference appends the failed pass-1 keypoints after the others) does not change the result.
// Not handled: fisheye calibrations (the device projection is the pinhole / radial-tangential model): a diagnostic, and the frame
// is left as it was.  Without a CUDA device every keypoint is lost, as the drop-in fbKltTracking reports it.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "visual_front_end.hpp"       // the reference's, unchanged
#include "feature_tracker.hpp"        // the drop-in class (host/feature_tracker.hpp): klt_convg_crit_
#include "abi_flat.hpp"
#include "pyr_cache.hpp"
#include "../../include/ov2b200.h"

void VisualFrontEnd::kltTracking()
{
    auto& frame = *pcurframe_;
    std::vector<int> ids;
    ids.reserve(frame.mapkps_.size());
    for (const auto& it : frame.mapkps_) ids.push_back(it.first);
    if (ids.empty()) return;
    auto cal = frame.pcalib_leftcam_;
    if (cal->model_ != CameraCalibration::Pinhole) {
        fprintf(stderr, "[ov2b200] kltTracking: only the pinhole (radial-tangential) model is built; keep the reference's body for fisheye\n");
        return;
    }
    ov2shim::DeviceState& s = ov2shim::device_state();
    ov2_pyr* dprev = nullptr;
    ov2_pyr* dcur = nullptr;
    const int nlev_extra = (int)prev_pyr_.size() / 2 - 1;
    if (s.ctx && !prev_pyr_.empty() && !cur_pyr_.empty()) {
        dprev = s.cache.get(s.ctx, prev_pyr_[0], nlev_extra);
        dcur = dprev ? s.cache.get(s.ctx, cur_pyr_[0], nlev_extra) : nullptr;
    }
    const int n = (int)ids.size();
    std::vector<float> px(2 * (size_t)n), tracked(2 * (size_t)n);
    std::vector<double> wpt(3 * (size_t)n, 0.0);
    std::vector<uint8_t> is3d(n, 0), status(n, 0), pass(n, 0);
    for (int i = 0; i < n; ++i) {
        const Keypoint& kp = frame.mapkps_.at(ids[i]);
        px[2 * i] = kp.px_.x;
        px[2 * i + 1] = kp.px_.y;
        if (kp.is3d_) {
            auto it = pmap_->map_plms_.find(kp.lmid_);
            if (it != pmap_->map_plms_.end() && it->second) {   // the reference's map_plms_.at() would throw here
                const Eigen::Vector3d w = it->second->getPoint();
                wpt[3 * i] = w.x(); wpt[3 * i + 1] = w.y(); wpt[3 * i + 2] = w.z();
                is3d[i] = 1;
            }
        }
    }
    uint8_t p3p = 0;
    int32_t nbgood = 0, nbkps = 0;
    ov2_status st = OV2_ERR_NO_DEVICE;
    if (dprev && dcur) {
        double T[12], K[4], D[5];
        ov2shim::put_pose(frame.getTcw(), T);
        const double* dist = ov2shim::put_pinhole(*cal, K, D);
        const int32_t wh[2] = {(int32_t)cal->img_w_, (int32_t)cal->img_h_};
        const int32_t offsets[2] = {0, n};
        ov2_klt_params prm;
        prm.win = pslamstate_->nklt_win_size_;
        prm.max_iter = ptracker_->klt_convg_crit_.maxCount;
        prm.eps = (float)ptracker_->klt_convg_crit_.epsilon;
        prm.ferr = (float)pslamstate_->nklt_err_;
        prm.fb_dist = pslamstate_->fmax_fbklt_dist_;
        st = ov2_klt_tracking(s.ctx, dprev, dcur, &prm, 0, 1, offsets, T, K, dist, wh, px.data(),
                              wpt.data(), is3d.data(), pslamstate_->nklt_pyr_lvl_, pslamstate_->klt_use_prior_ ? 1 : 0,
                              tracked.data(), status.data(), pass.data(), &p3p, &nbgood, &nbkps);
    }
    if (st != OV2_OK) {
        fprintf(stderr, "[ov2b200] kltTracking: %s\n", s.ctx ? ov2_last_error(s.ctx) : "no CUDA device (no CPU fallback)");
        for (int i = 0; i < n; ++i) pmap_->removeObsFromCurFrameById(ids[i]);
        return;
    }
    // visual_front_end.cpp:201-209, 228-233, 248-258
    for (int i = 0; i < n; ++i)
        if (pass[i] == 1) frame.updateKeypoint(ids[i], cv::Point2f(tracked[2 * i], tracked[2 * i + 1]));
    if (p3p) bp3preq_ = true;
    for (int i = 0; i < n; ++i) {
        if (pass[i] == 1) continue;
        if (status[i]) frame.updateKeypoint(ids[i], cv::Point2f(tracked[2 * i], tracked[2 * i + 1]));
        else pmap_->removeObsFromCurFrameById(ids[i]);
    }
}
