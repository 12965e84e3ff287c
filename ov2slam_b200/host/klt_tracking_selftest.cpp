// Drives the drop-in VisualFrontEnd::kltTracking (host/visual_front_end_klt_gpu.cpp) the way VisualFrontEnd::trackMono does
// (/root/reference/src/visual_front_end.cpp:104) on a SYNTHETIC frame: reads the keypoints (id, 3-D flag, pixel, map point), the
// calibration, the pose and the two images written by tests/test_klt_tracking_shim.py, builds the frame and the map with the stand-in
// classes (host/standin/ref/), hands in the two pyramid vectors (entry 0 = the image; the drop-ins read only that entry and the
// vector's length), calls kltTracking and writes what it left in the frame.
//
//   klt_tracking_selftest scene.bin result.bin
// scene.bin:  i32 n, w, h, use_prior, win, nklt_pyr_lvl, has_dist; f64 K[4], D[4], Twc[7] (tx ty tz qx qy qz qw);
//             per keypoint: i32 lmid, is3d; f32 px[2]; f64 wpt[3]; then the previous and the current image (w * h bytes each)
// result.bin: i32 n; f64 Tcw[12] (the pose as the drop-in flattens it); i32 bp3preq;
//             per keypoint in scene order: i32 lmid, alive; f32 px[2]
#include <cstdio>
#include <cstring>
#include <vector>

#include "visual_front_end.hpp"
#include "feature_tracker.hpp"
#include "abi_flat.hpp"

struct KpRec { int32_t lmid, is3d; float px[2]; double wpt[3]; };

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: klt_tracking_selftest scene.bin result.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hd[7];
    double K[4], D[4], Twc[7];
    if (fread(hd, 4, 7, f) != 7 || fread(K, 8, 4, f) != 4 || fread(D, 8, 4, f) != 4 || fread(Twc, 8, 7, f) != 7) return 3;
    const int n = hd[0], w = hd[1], h = hd[2];
    std::vector<KpRec> recs(n);
    for (auto& r : recs)
        if (fread(&r.lmid, 4, 2, f) != 2 || fread(r.px, 4, 2, f) != 2 || fread(r.wpt, 8, 3, f) != 3) return 3;
    cv::Mat im0(h, w, CV_8UC1), im1(h, w, CV_8UC1);
    if (fread(im0.data, 1, (size_t)w * h, f) != (size_t)w * h || fread(im1.data, 1, (size_t)w * h, f) != (size_t)w * h) return 3;
    fclose(f);

    auto params = std::make_shared<SlamParams>();
    params->klt_use_prior_ = hd[3] != 0;
    params->nklt_win_size_ = hd[4];
    params->nklt_pyr_lvl_ = hd[5];
    auto cal = std::make_shared<CameraCalibration>();
    cal->setK(K[0], K[1], K[2], K[3]);
    cal->img_w_ = w; cal->img_h_ = h;
    if (hd[6]) {
        cal->k1_ = D[0]; cal->k2_ = D[1]; cal->p1_ = D[2]; cal->p2_ = D[3];
        cal->Dcv_ = cv::Mat(1, 4, CV_8UC1);                  // non-empty: the calibration has a distortion model
    }
    auto frame = std::make_shared<Frame>();
    frame->pcalib_leftcam_ = cal;
    frame->setTwc(Sophus::SE3d(Eigen::Quaterniond(Twc[6], Twc[3], Twc[4], Twc[5]), Eigen::Vector3d(Twc[0], Twc[1], Twc[2])));
    auto map = std::make_shared<MapManager>();
    map->pcurframe_ = frame;
    for (const auto& r : recs) {
        Keypoint kp;
        kp.lmid_ = r.lmid; kp.is3d_ = r.is3d != 0;
        kp.px_ = cv::Point2f(r.px[0], r.px[1]);
        frame->mapkps_[kp.lmid_] = kp;
        if (kp.is3d_) {
            auto lm = std::make_shared<MapPoint>();
            lm->lmid_ = r.lmid;
            lm->ptxyz_ = Eigen::Vector3d(r.wpt[0], r.wpt[1], r.wpt[2]);
            map->map_plms_[r.lmid] = lm;
        }
    }
    VisualFrontEnd fe;
    fe.pslamstate_ = params;
    fe.pcurframe_ = frame;
    fe.pmap_ = map;
    fe.ptracker_ = std::make_shared<FeatureTracker>(30, 0.01f, nullptr);
    for (int lv = 0, lw = w, lh = h; lv <= params->nklt_pyr_lvl_; ++lv, lw = (lw + 1) / 2, lh = (lh + 1) / 2) {
        fe.prev_pyr_.push_back(lv == 0 ? im0 : cv::Mat(lh, lw, CV_8UC1));
        fe.prev_pyr_.push_back(cv::Mat());
        fe.cur_pyr_.push_back(lv == 0 ? im1 : cv::Mat(lh, lw, CV_8UC1));
        fe.cur_pyr_.push_back(cv::Mat());
    }

    fe.kltTracking();

    FILE* g = fopen(argv[2], "wb");
    if (!g) return 4;
    double T[12];
    ov2shim::put_pose(frame->getTcw(), T);
    int32_t v = n;
    fwrite(&v, 4, 1, g);
    fwrite(T, 8, 12, g);
    v = fe.bp3preq_ ? 1 : 0;
    fwrite(&v, 4, 1, g);
    int alive_n = 0;
    for (const auto& r : recs) {
        auto it = frame->mapkps_.find(r.lmid);
        const int32_t rec[2] = {r.lmid, it != frame->mapkps_.end() ? 1 : 0};
        const float p[2] = {rec[1] ? it->second.px_.x : -1.f, rec[1] ? it->second.px_.y : -1.f};
        alive_n += rec[1];
        fwrite(rec, 4, 2, g);
        fwrite(p, 4, 2, g);
    }
    fclose(g);
    printf("kltTracking: %d keypoints, %d tracked, bp3preq %d\n", n, alive_n, fe.bp3preq_ ? 1 : 0);
    return 0;
}
