// Drives the drop-in MapManager::stereoMatching (host/map_manager_stereo_gpu.cpp) the way Mapper::run does for a new stereo
// keyframe (/root/reference/src/mapper.cpp:75-81) on a SYNTHETIC keyframe: reads the keypoints (pixel, undistorted pixel, bearing,
// 3-D flag, map point or none) and the rig written by tests/test_host_shim.py, builds the frame, its grid and the map with the
// stand-in classes (host/standin/ref/map_manager.hpp), hands in blank image pyramids of the right shapes, calls stereoMatching and
// writes which keypoints became stereo keypoints and with which right pixel.
//
//   stereo_selftest scene.bin result.bin [disparity]
// With a disparity, the images are a smooth synthetic texture and its copy shifted by that many pixels (a fronto-parallel plane for a
// rectified rig) instead of blank images: the GPU test checks that the stereo keypoints land `disparity` pixels to the left.
// scene.bin: i32 nkps, rect, w, h, ncellsize, nbwcells, ncells; f64 K[4], Kr[4], Tc0c1[7] (tx ty tz qx qy qz qw), Twc[7], Frl[9];
//            per keypoint: i32 lmid, i32 is3d, i32 has_mp; f32 px[2], unpx[2]; f64 bv[3], wpt[3];
//            optionally f64 Dr[4] (k1 k2 p1 p2 of the right camera; absent or all zero: no distortion model)
// result.bin: i32 nkps, order[nkps] (the lmids as Frame::getKeypoints() returned them - the order of all the lists);
//             per keypoint in that order: i32 is_stereo, f32 rpx[2]; i32 n_removed_obs;
//             f64 Tcw[12], Trl[12] (the keyframe's pose and the rig as the drop-in flattens them)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "map_manager.hpp"
#include "feature_tracker.hpp"
#include "abi_flat.hpp"

struct KpRec { int32_t lmid, is3d, has_mp; float px[2], unpx[2]; double bv[3], wpt[3]; };

static Sophus::SE3d se3_of(const double* p) {
    return Sophus::SE3d(Eigen::Quaterniond(p[6], p[3], p[4], p[5]), Eigen::Vector3d(p[0], p[1], p[2]));
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: stereo_selftest scene.bin result.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hd[7];
    double K[4], Kr[4], Dr[4] = {0, 0, 0, 0}, Trig[7], Twc[7], Frl[9];
    if (fread(hd, 4, 7, f) != 7 || fread(K, 8, 4, f) != 4 || fread(Kr, 8, 4, f) != 4 || fread(Trig, 8, 7, f) != 7 || fread(Twc, 8, 7, f) != 7 ||
        fread(Frl, 8, 9, f) != 9)
        return 3;
    const int nkps = hd[0], w = hd[2], h = hd[3], cs = hd[4], nbw = hd[5], ncells = hd[6];
    std::vector<KpRec> recs(nkps);
    for (auto& r : recs)
        if (fread(&r.lmid, 4, 3, f) != 3 || fread(r.px, 4, 4, f) != 4 || fread(r.bv, 8, 6, f) != 6) return 3;
    if (fread(Dr, 8, 4, f) != 4 && ferror(f)) return 3;
    fclose(f);

    auto params = std::make_shared<SlamParams>();
    params->stereo_ = true;
    params->bdo_stereo_rect_ = hd[1] != 0;
    auto map = std::make_shared<MapManager>();
    map->pslamstate_ = params;
    map->ptracker_ = std::make_shared<FeatureTracker>(30, 0.01f, nullptr);
    auto lcal = std::make_shared<CameraCalibration>(), rcal = std::make_shared<CameraCalibration>();
    lcal->setK(K[0], K[1], K[2], K[3]); lcal->img_w_ = w; lcal->img_h_ = h;
    rcal->setK(Kr[0], Kr[1], Kr[2], Kr[3]); rcal->img_w_ = w; rcal->img_h_ = h;
    if (Dr[0] != 0 || Dr[1] != 0 || Dr[2] != 0 || Dr[3] != 0) {
        rcal->k1_ = Dr[0]; rcal->k2_ = Dr[1]; rcal->p1_ = Dr[2]; rcal->p2_ = Dr[3];
        rcal->Dcv_ = cv::Mat(1, 4, CV_8UC1);                  // non-empty: the calibration has a distortion model
    }
    rcal->Tc0ci_ = se3_of(Trig);
    rcal->Tcic0_ = rcal->Tc0ci_.inverse();
    Frame frame;
    frame.id_ = frame.kfid_ = 7;
    frame.pcalib_leftcam_ = lcal; frame.pcalib_rightcam_ = rcal;
    frame.setTwc(se3_of(Twc));
    memcpy(frame.Frl_.m, Frl, sizeof(Frl));
    frame.ncellsize_ = cs; frame.nbwcells_ = nbw; frame.nbhcells_ = ncells / nbw;
    frame.vgridkps_.resize(ncells);
    for (const auto& r : recs) {
        Keypoint kp;
        kp.lmid_ = r.lmid; kp.is3d_ = r.is3d != 0;
        kp.px_ = cv::Point2f(r.px[0], r.px[1]); kp.unpx_ = cv::Point2f(r.unpx[0], r.unpx[1]);
        kp.bv_ = Eigen::Vector3d(r.bv[0], r.bv[1], r.bv[2]);
        frame.mapkps_[kp.lmid_] = kp;
        frame.nbkps_++;
        if (kp.is3d_) frame.nb3dkps_++; else frame.nb2dkps_++;
        const int cell = (int)std::floor(kp.px_.y / cs) * nbw + (int)std::floor(kp.px_.x / cs);
        if (cell >= 0 && cell < ncells) frame.vgridkps_[cell].push_back(kp.lmid_);
        if (r.has_mp) {
            auto lm = std::make_shared<MapPoint>();
            lm->lmid_ = r.lmid; lm->is3d_ = kp.is3d_;
            lm->ptxyz_ = Eigen::Vector3d(r.wpt[0], r.wpt[1], r.wpt[2]);
            map->map_plms_[r.lmid] = lm;
        }
    }
    // image pyramids as the reference keeps them: (image, derivative) pairs per level; the pixels are irrelevant to the flow
    std::vector<cv::Mat> lpyr, rpyr;
    for (int lv = 0, lw = w, lh = h; lv <= params->nklt_pyr_lvl_; ++lv, lw = (lw + 1) / 2, lh = (lh + 1) / 2) {
        for (int side = 0; side < 2; ++side) {
            cv::Mat im(lh, lw, CV_8UC1);
            memset(im.data, 40 + 17 * side + lv, (size_t)lw * lh);
            if (argc > 3 && lv == 0) {
                const double shift = side ? atof(argv[3]) : 0.0;
                for (int y = 0; y < lh; ++y)
                    for (int x = 0; x < lw; ++x) {
                        const double u = x + shift;
                        const double v = 128 + 50 * std::sin(0.11 * u + 0.07 * y) + 40 * std::sin(0.05 * u - 0.13 * y + 1) + 30 * std::sin(0.31 * u + 0.23 * y + 2);
                        im.ptr(y)[x] = (unsigned char)std::lrint(v);
                    }
            }
            (side ? rpyr : lpyr).push_back(im);
            (side ? rpyr : lpyr).push_back(cv::Mat());
        }
    }
    std::vector<int32_t> order;
    for (const auto& kp : frame.getKeypoints()) order.push_back(kp.lmid_);

    map->stereoMatching(frame, lpyr, rpyr);

    FILE* g = fopen(argv[2], "wb");
    if (!g) return 4;
    int32_t n = nkps;
    fwrite(&n, 4, 1, g); fwrite(order.data(), 4, order.size(), g);
    int nstereo = 0;
    for (const int id : order) {
        const Keypoint kp = frame.getKeypointById(id);
        int32_t st = kp.is_stereo_ ? 1 : 0;
        float rp[2] = {kp.rpx_.x, kp.rpx_.y};
        nstereo += st;
        fwrite(&st, 4, 1, g); fwrite(rp, 4, 2, g);
    }
    n = (int32_t)map->removed_obs_.size();
    fwrite(&n, 4, 1, g);
    double T[24];
    ov2shim::put_pose(frame.getTcw(), T);
    ov2shim::put_pose(rcal->Tcic0_, T + 12);
    fwrite(T, 8, 24, g);
    fclose(g);
    printf("stereoMatching: %d keypoints, %d stereo, %d observations dropped\n", nkps, nstereo, n);
    return 0;
}
