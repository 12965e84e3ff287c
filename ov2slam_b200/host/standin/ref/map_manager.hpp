// Minimal STAND-INS for the map classes Optimizer::localBA reads and writes (the reference's include/map_manager.hpp,
// frame.hpp, map_point.hpp, camera_calibration.hpp, slam_params.hpp): same member / method names and signatures for the
// subset the shim uses, trivial in-memory implementations.  Only for compile-checking and self-testing
// ov2slam_b200/host/optimizer_localba_gpu.cpp in a container without the reference's dependencies (ROS, PCL, OpenCV,
// Eigen, Sophus); on a box that builds the reference, its own headers are used instead.
#pragma once
#include <cmath>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <unordered_map>
#include <vector>

#include <opencv2/core.hpp>
#include <sophus/se3.hpp>

class FeatureTracker;   // the drop-in class of host/feature_tracker.hpp (the reference's include/feature_tracker.hpp)

struct SlamParams {
    int nmin_covscore_ = 25;
    int nklt_pyr_lvl_ = 3, nklt_win_size_ = 9, nklt_err_ = 30;
    float fmax_fbklt_dist_ = 0.5f;
    bool bdo_stereo_rect_ = false, debug_ = false, log_timings_ = false, klt_use_prior_ = true;
    bool stereo_ = false, buse_inv_depth_ = true, apply_l2_after_robust_ = true;
    float robust_mono_th_ = 5.9915f;
};

class CameraCalibration {
public:
    enum Model { Pinhole, Fisheye };
    Model model_ = Pinhole;
    double fx_ = 0, fy_ = 0, cx_ = 0, cy_ = 0;
    double k1_ = 0, k2_ = 0, p1_ = 0, p2_ = 0;
    double img_w_ = 0, img_h_ = 0;
    cv::Mat Dcv_;                                       // empty: no distortion (camera_calibration.cpp:262)
    Eigen::Matrix3d iK_;
    Sophus::SE3d Tc0ci_, Tcic0_;                        // the reference keeps Tcic0_ = Tc0ci_.inverse() (camera_calibration.cpp:197-198)
    void setK(double fx, double fy, double cx, double cy) {
        fx_ = fx; fy_ = fy; cx_ = cx; cy_ = cy;
        iK_ = Eigen::Matrix3d();
        iK_.m[0] = 1.0 / fx; iK_.m[2] = -cx / fx; iK_.m[4] = 1.0 / fy; iK_.m[5] = -cy / fy;
    }
    Sophus::SE3d getExtrinsic() const { return Tc0ci_; }
    // stand-in calibrations carry no distortion model on this path (rectified / undistorted images)
    cv::Point2f undistortImagePoint(const cv::Point2f& pt) const { return pt; }
    cv::Point2f projectCamToImageDist(const Eigen::Vector3d& pt) const {
        return cv::Point2f((float)(fx_ * pt.x() / pt.z() + cx_), (float)(fy_ * pt.y() / pt.z() + cy_));
    }
    // rectification (camera_calibration.hpp:67,116,120): the maps setUndistStereoMap / setUndistMap build, and the lock
    // rectifyImage takes; the body is the drop-in of host/camera_calibration_rect_gpu.cpp
    void rectifyImage(const cv::Mat& img, cv::Mat& rect) const;
    cv::Mat undist_map_x_, undist_map_y_;
    mutable std::mutex intrinsic_mutex_, extrinsic_mutex_;
};

struct Keypoint {
    int lmid_ = -1;
    cv::Point2f px_;
    cv::Point2f unpx_, runpx_, rpx_;
    Eigen::Vector3d bv_;
    int scale_ = 0;
    bool is3d_ = false, is_stereo_ = false;
};

class Frame {
public:
    int id_ = 0, kfid_ = 0;
    size_t nbkps_ = 0, nb2dkps_ = 0, nb3dkps_ = 0, nb_stereo_kps_ = 0;
    std::shared_ptr<CameraCalibration> pcalib_leftcam_, pcalib_rightcam_;
    std::unordered_map<int, Keypoint> mapkps_;
    std::vector<std::vector<int>> vgridkps_;            // keypoint (= map point) ids per grid cell, insertion order
    size_t ncellsize_ = 35, nbwcells_ = 0, nbhcells_ = 0;
    std::map<int, int> covkfs_;
    Sophus::SE3d Twc_;

    std::vector<Keypoint> getKeypoints() const {
        std::vector<Keypoint> v;
        for (const auto& kv : mapkps_) v.push_back(kv.second);
        return v;
    }
    bool isObservingKp(const int lmid) const { return mapkps_.count(lmid) != 0; }
    std::vector<Keypoint> getKeypoints3d() const {
        std::vector<Keypoint> v;
        for (const auto& kv : mapkps_) if (kv.second.is3d_) v.push_back(kv.second);
        return v;
    }
    Keypoint getKeypointById(const int lmid) const { auto it = mapkps_.find(lmid); return it == mapkps_.end() ? Keypoint() : it->second; }
    void removeStereoKeypointById(const int lmid) { auto it = mapkps_.find(lmid); if (it != mapkps_.end()) it->second.is_stereo_ = false; }
    Sophus::SE3d getTcw() const { return Twc_.inverse(); }
    Eigen::Vector3d projWorldToCam(const Eigen::Vector3d& wpt) const { return Twc_.inverse() * wpt; }
    // ---- what MapManager::stereoMatching reads and writes (frame.cpp:423-433, 594-622, 830-870)
    Eigen::Matrix3d Frl_;
    cv::Point2f projCamToRightImageDist(const Eigen::Vector3d& pt) const {
        return pcalib_rightcam_->projectCamToImageDist(pcalib_rightcam_->Tcic0_ * pt);
    }
    cv::Point2f projWorldToRightImageDist(const Eigen::Vector3d& wpt) const { return projCamToRightImageDist(projWorldToCam(wpt)); }
    bool isInRightImage(const cv::Point2f& pt) const {
        return pt.x >= 0 && pt.y >= 0 && pt.x < pcalib_rightcam_->img_w_ && pt.y < pcalib_rightcam_->img_h_;
    }
    std::vector<Keypoint> getSurroundingKeypoints(const Keypoint& kp) const {
        std::vector<Keypoint> vkps;
        const int rkp = (int)std::floor(kp.px_.y / ncellsize_), ckp = (int)std::floor(kp.px_.x / ncellsize_);
        for (int r = rkp - 1; r < rkp + 1; r++)
            for (int c = ckp - 1; c < ckp + 1; c++) {
                const int idx = r * (int)nbwcells_ + c;
                if (r < 0 || c < 0 || idx >= (int)vgridkps_.size()) continue;
                for (const int id : vgridkps_[idx])
                    if (id != kp.lmid_) { auto it = mapkps_.find(id); if (it != mapkps_.end()) vkps.push_back(it->second); }
            }
        return vkps;
    }
    void updateKeypointStereo(const int lmid, const cv::Point2f& pt) {
        auto it = mapkps_.find(lmid);
        if (it == mapkps_.end()) return;
        it->second.rpx_ = pt;
        it->second.runpx_ = pcalib_rightcam_->undistortImagePoint(pt);
        if (!it->second.is_stereo_) { it->second.is_stereo_ = true; nb_stereo_kps_++; }
    }
    // Frame::updateKeypoint(lmid, pt) (frame.cpp:334-370): the stand-in moves the pixel only (the reference also refreshes the
    // undistorted pixel, the bearing and the grid cell)
    void updateKeypoint(const int lmid, const cv::Point2f& pt) { auto it = mapkps_.find(lmid); if (it != mapkps_.end()) it->second.px_ = pt; }
    Sophus::SE3d getTwc() const { return Twc_; }
    void setTwc(const Sophus::SE3d& Twc) { Twc_ = Twc; }
    std::map<int, int> getCovisibleKfMap() const { return covkfs_; }
    void removeCovisibleKf(const int kfid) { covkfs_.erase(kfid); }
};

class MapPoint {
public:
    int lmid_ = -1, kfid_ = -1;
    bool isobs_ = true, bad_ = false, is3d_ = true;
    double invdepth_ = -1;
    cv::Mat desc_;                                      // the map point's representative descriptor (1 x 32, 8-bit)
    std::unordered_map<int, cv::Mat> map_kf_desc_;      // one descriptor per observing keyframe
    Eigen::Vector3d ptxyz_;
    std::set<int> set_kfids_;
    bool isBad() const { return bad_; }
    std::set<int> getKfObsSet() const { return set_kfids_; }
    Eigen::Vector3d getPoint() const { return ptxyz_; }
};

class MapManager {
public:
    std::unordered_map<int, std::shared_ptr<Frame>> map_pkfs_;
    std::unordered_map<int, std::shared_ptr<MapPoint>> map_plms_;
    std::shared_ptr<Frame> pcurframe_;
    std::shared_ptr<SlamParams> pslamstate_;
    std::shared_ptr<FeatureTracker> ptracker_;
    void stereoMatching(Frame &frame, const std::vector<cv::Mat> &vleftpyr, const std::vector<cv::Mat> &vrightpyr);   // map_manager.hpp:83
    int nkfid_ = 0;                                     // id of the newest keyframe
    std::mutex map_mutex_, optim_mutex_;
    std::vector<std::pair<int, int>> removed_obs_;      // (lmid, kfid) - for the self-test's report
    std::vector<int> removed_points_;

    std::shared_ptr<Frame> getKeyframe(const int kfid) const { auto it = map_pkfs_.find(kfid); return it == map_pkfs_.end() ? nullptr : it->second; }
    std::shared_ptr<MapPoint> getMapPoint(const int lmid) const { auto it = map_plms_.find(lmid); return it == map_plms_.end() ? nullptr : it->second; }
    void removeMapPointObs(const int lmid, const int kfid) {
        removed_obs_.emplace_back(lmid, kfid);
        auto lm = getMapPoint(lmid);
        if (lm) lm->set_kfids_.erase(kfid);
        auto kf = getKeyframe(kfid);
        if (kf) kf->mapkps_.erase(lmid);
    }
    void removeObsFromCurFrameById(const int lmid) { if (pcurframe_) pcurframe_->mapkps_.erase(lmid); }
    void removeMapPoint(const int lmid) { removed_points_.push_back(lmid); map_plms_.erase(lmid); }
    void updateMapPoint(const int lmid, const Eigen::Vector3d& wpt, const double kfanch_invdepth = -1.) {
        auto lm = getMapPoint(lmid);
        if (!lm) return;
        lm->ptxyz_ = wpt;
        if (kfanch_invdepth >= 0.) lm->invdepth_ = kfanch_invdepth;
    }
};
