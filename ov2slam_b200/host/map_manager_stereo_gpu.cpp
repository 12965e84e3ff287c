// MapManager::stereoMatching on the GPU (8f-3): the reference's declaration (include/map_manager.hpp:83) is kept, this translation
// unit supplies the body of /root/reference/src/map_manager.cpp:367-611.  Exclude the reference's own body with
// #ifndef OV2_EXTERNAL_STEREOMATCHING.
//
// It flattens the keyframe's keypoints (frame.getKeypoints(), in that order) with their map points, the pose, the right
// calibration, the rig and, for rigs that are not rectified, the grid; reads the two pyramids from the device-pyramid cache
// (pyr_cache.hpp) and makes ONE ov2_stereo_matching call: the priors, the row search, the two tracker passes, the undistortion and
// the epipolar gate run on the device without a synchronisation between them.  Then every stereo match becomes
// updateKeypointStereo.  3-D keypoints whose map point is gone lose their observation while flattening (:411-414), as in the
// reference; the device drops them.
// Not handled: fisheye right calibrations (the device projection is the pinhole / radial-tangential model): a diagnostic, and the
// frame and the map are left as they were.  Without a CUDA device no keypoint becomes a stereo keypoint.
// Compile-checked and self-tested against the stand-in map classes (host/standin/ref/): host/stereo_selftest.cpp.
#include <cstdint>
#include <iostream>
#include <vector>

#include "map_manager.hpp"             // the reference's, unchanged
#include "feature_tracker.hpp"         // the drop-in class (host/feature_tracker.hpp): klt_convg_crit_
#include "abi_flat.hpp"
#include "pyr_cache.hpp"
#include "../../include/ov2b200.h"

void MapManager::stereoMatching(Frame &frame, const std::vector<cv::Mat> &vleftpyr, const std::vector<cv::Mat> &vrightpyr)
{
    const SlamParams& cfg = *pslamstate_;
    const bool rectified = cfg.bdo_stereo_rect_;
    const int nlvl = cfg.nklt_pyr_lvl_;                          // pyramid level of the row search (entry 2 * level of the vectors)
    if (rectified && (vleftpyr.size() <= (size_t)(2 * nlvl) || vrightpyr.size() <= (size_t)(2 * nlvl))) {
        std::cerr << "[ov2b200] stereoMatching: the pyramids have no level " << nlvl << " for the row search\n";
        return;
    }
    const auto cal = frame.pcalib_rightcam_;
    if (cal->model_ != CameraCalibration::Pinhole) {
        std::cerr << "[ov2b200] stereoMatching: only the pinhole (radial-tangential) model is built; keep the reference's body for fisheye\n";
        return;
    }
    const std::vector<Keypoint> vkps = frame.getKeypoints();
    const int n = (int)vkps.size();
    std::vector<float> px(2 * (size_t)n), unpx(2 * (size_t)n), right(2 * (size_t)n);
    std::vector<double> bv(3 * (size_t)n), wpt(3 * (size_t)n, 0.0);
    std::vector<uint8_t> is3d(n, 0), has_mp(n, 0), stereo(n, 0), pass(n, 0);
    for (int i = 0; i < n; ++i) {
        const Keypoint& kp = vkps[i];
        px[2 * i] = kp.px_.x; px[2 * i + 1] = kp.px_.y;
        unpx[2 * i] = kp.unpx_.x; unpx[2 * i + 1] = kp.unpx_.y;
        bv[3 * i] = kp.bv_.x(); bv[3 * i + 1] = kp.bv_.y(); bv[3 * i + 2] = kp.bv_.z();
        if (!kp.is3d_) continue;
        is3d[i] = 1;
        const auto plm = getMapPoint(kp.lmid_);
        if (plm == nullptr) { removeMapPointObs(kp.lmid_, frame.kfid_); continue; }
        has_mp[i] = 1;
        const Eigen::Vector3d w = plm->getPoint();
        wpt[3 * i] = w.x(); wpt[3 * i + 1] = w.y(); wpt[3 * i + 2] = w.z();
    }
    std::vector<int32_t> cell_ptr, cell_kps;
    if (!rectified && !ov2shim::grid_csr(frame, vkps, "stereoMatching", cell_ptr, cell_kps)) return;
    const int32_t cell_offsets[2] = {0, (int32_t)frame.vgridkps_.size()};
    const int32_t grid[2] = {(int32_t)frame.ncellsize_, (int32_t)frame.nbwcells_};
    const int32_t offsets[2] = {0, n};
    const int32_t wh[2] = {(int32_t)cal->img_w_, (int32_t)cal->img_h_};
    double Tcw[12], Trl[12], Frl[9], K[4], D[5];
    ov2shim::put_pose(frame.getTcw(), Tcw);
    ov2shim::put_pose(cal->Tcic0_, Trl);                         // what Frame::projCamToRightImageDist applies (frame.cpp:796-799)
    ov2shim::put_mat3(frame.Frl_, Frl);
    const double* dist = ov2shim::put_pinhole(*cal, K, D);
    ov2_klt_params prm;
    prm.win = cfg.nklt_win_size_;
    prm.max_iter = ptracker_->klt_convg_crit_.maxCount;
    prm.eps = (float)ptracker_->klt_convg_crit_.epsilon;
    prm.ferr = (float)cfg.nklt_err_;
    prm.fb_dist = cfg.fmax_fbklt_dist_;

    ov2shim::DeviceState& s = ov2shim::device_state();
    int32_t nstereo = 0;
    ov2_status st = n == 0 ? OV2_OK : OV2_ERR_NO_DEVICE;
    if (n > 0 && s.ctx && !vleftpyr.empty() && !vrightpyr.empty()) {
        const int nlev_extra = (int)vleftpyr.size() / 2 - 1;
        ov2_pyr* dleft = s.cache.get(s.ctx, vleftpyr[0], nlev_extra);
        ov2_pyr* dright = dleft ? s.cache.get(s.ctx, vrightpyr[0], nlev_extra) : nullptr;
        st = dright ? ov2_stereo_matching(s.ctx, dleft, dright, &prm, 0, 1, offsets, Tcw, K, dist, Trl, Frl, wh,
                                          rectified ? nullptr : cell_offsets, rectified ? nullptr : grid,
                                          rectified ? nullptr : cell_ptr.data(), rectified ? nullptr : cell_kps.data(), px.data(),
                                          unpx.data(), bv.data(), is3d.data(), has_mp.data(), wpt.data(), rectified ? 1 : 0, nlvl,
                                          right.data(), stereo.data(), pass.data(), &nstereo)
                    : OV2_ERR_CUDA;
    }
    if (st != OV2_OK) {
        std::cerr << "[ov2b200] stereoMatching: " << (s.ctx ? ov2_last_error(s.ctx) : "no CUDA device (no CPU fallback)") << "\n";
        return;
    }
    // map_manager.cpp:575-604.  Each call touches one keypoint id, so the order (the reference's: pass-1 tracks first) does not
    // change the result.
    for (int i = 0; i < n; ++i)
        if (stereo[i]) frame.updateKeypointStereo(vkps[i].lmid_, cv::Point2f(right[2 * i], right[2 * i + 1]));
    if (cfg.debug_) std::cout << "\n \t>>> Nb of stereo tracks: " << nstereo << "\n";
}
