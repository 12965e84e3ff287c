// Drives the drop-in Optimizer::localBA (host/optimizer_localba_gpu.cpp) the way Estimator::applyLocalBA does
// (/root/reference/src/estimator.cpp:67-98) on a SYNTHETIC map: reads a flat window written by
// tests/test_host_shim.py, builds keyframes / map points / covisibility from it (stand-in map classes,
// host/standin/ref/map_manager.hpp), calls localBA, and writes the keyframe poses and landmark inverse depths the map
// holds afterwards.  The test compares them with ov2_localba_solve on the flat window (what the Python binding runs).
//
//   optimizer_selftest window.bin result.bin [stop]
// window.bin: int32 ncam, npts, nobs, stereo; f64 K[4], Kr[4], Trl[7]; f64 pose[ncam][7]; u8 pose_const[ncam];
//             i32 lm_anchor_cam[npts]; f64 lm_anchor_px[npts][2]; f64 lm_invdepth[npts]; i32 obs_cam[nobs]; i32 obs_lm[nobs];
//             f64 obs_px[nobs][2]; u8 obs_type[nobs]
// result.bin: f64 pose[ncam][7]; f64 invdepth[npts] (-1: map point removed); i32 n_removed_obs
//
//   optimizer_selftest pnp problem.bin result.bin
// Calls both MultiViewGeometry::ceresPnP overloads (host/multi_view_geometry_pnp_gpu.cpp), the way VisualFrontEnd::computePose
// and LoopCloser call them, on one pose problem.
// problem.bin: i32 n, nmaxiter, use_robust, apply_l2; f32 chi2th, fx, fy, cx, cy; f64 Twc[7] (t, q xyzw); f64 unpx[n][2];
//              f64 wpts[n][3]; i32 scales[n]
// result.bin:  per overload (first with the scales, then the scale-less one): i32 return value; f64 Twc[7] as the call left it;
//              i32 nout; i32 voutliersidx[nout]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "multi_view_geometry.hpp"
#include "optimizer.hpp"

void Optimizer::signalStopLocalBA() { bstop_localba_ = true; }      // the reference's optimizer.cpp:2334-2343
bool Optimizer::stopLocalBA() { return bstop_localba_; }

template <typename T> static bool rd(FILE* f, std::vector<T>& v, size_t n) { v.resize(n); return n == 0 || fread(v.data(), sizeof(T), n, f) == n; }

static int pnp_main(const char* in, const char* outp) {
    FILE* f = fopen(in, "rb");
    if (!f) return 3;
    int32_t hd[4];
    float fl[5];
    std::vector<double> T, px, wp;
    std::vector<int32_t> sc;
    if (fread(hd, 4, 4, f) != 4 || fread(fl, 4, 5, f) != 5) return 3;
    const size_t n = (size_t)hd[0];
    if (!rd(f, T, 7) || !rd(f, px, 2 * n) || !rd(f, wp, 3 * n) || !rd(f, sc, n)) return 3;
    fclose(f);
    std::vector<Eigen::Vector2d, Eigen::aligned_allocator<Eigen::Vector2d> > vunkps;
    std::vector<Eigen::Vector3d, Eigen::aligned_allocator<Eigen::Vector3d> > vwpts;
    for (size_t i = 0; i < n; ++i) {
        vunkps.emplace_back(px[2 * i], px[2 * i + 1]);
        vwpts.emplace_back(wp[3 * i], wp[3 * i + 1], wp[3 * i + 2]);
    }
    const std::vector<int> vscales(sc.begin(), sc.end());
    f = fopen(outp, "wb");
    if (!f) return 3;
    for (int overload = 0; overload < 2; ++overload) {
        Sophus::SE3d Twc(Eigen::Quaterniond(T[6], T[3], T[4], T[5]), Eigen::Vector3d(T[0], T[1], T[2]));
        std::vector<int> vout;
        const bool ok = overload == 0
            ? MultiViewGeometry::ceresPnP(vunkps, vwpts, vscales, Twc, hd[1], fl[0], hd[2] != 0, hd[3] != 0, fl[1], fl[2], fl[3], fl[4], vout)
            : MultiViewGeometry::ceresPnP(vunkps, vwpts, Twc, hd[1], fl[0], hd[2] != 0, hd[3] != 0, fl[1], fl[2], fl[3], fl[4], vout);
        const int32_t r = ok ? 1 : 0, nout = (int32_t)vout.size();
        const Eigen::Quaterniond& q = Twc.unit_quaternion();
        const double p[7] = {Twc.translation().x(), Twc.translation().y(), Twc.translation().z(), q.x(), q.y(), q.z(), q.w()};
        fwrite(&r, 4, 1, f);
        fwrite(p, sizeof(double), 7, f);
        fwrite(&nout, 4, 1, f);
        for (int i : vout) { const int32_t v = i; fwrite(&v, 4, 1, f); }
    }
    fclose(f);
    return 0;
}

int main(int argc, char** argv) {
    if (argc == 4 && std::string(argv[1]) == "pnp") return pnp_main(argv[2], argv[3]);
    if (argc < 3) { fprintf(stderr, "usage: optimizer_selftest window.bin result.bin [stop]\n       optimizer_selftest pnp problem.bin result.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 3;
    int32_t hd[4];
    if (fread(hd, 4, 4, f) != 4) return 3;
    const int ncam = hd[0], npts = hd[1], nobs = hd[2];
    const bool stereo = hd[3] != 0;
    std::vector<double> K, Kr, Trl, pose, apx, invd, opx;
    std::vector<uint8_t> pc, oty;
    std::vector<int32_t> lac, oc, ol;
    if (!rd(f, K, 4) || !rd(f, Kr, 4) || !rd(f, Trl, 7) || !rd(f, pose, 7 * (size_t)ncam) || !rd(f, pc, ncam) || !rd(f, lac, npts) ||
        !rd(f, apx, 2 * (size_t)npts) || !rd(f, invd, npts) || !rd(f, oc, nobs) || !rd(f, ol, nobs) || !rd(f, opx, 2 * (size_t)nobs) ||
        !rd(f, oty, nobs))
        return 3;
    fclose(f);
    auto params = std::make_shared<SlamParams>();
    params->stereo_ = stereo;
    auto map = std::make_shared<MapManager>();
    auto lcal = std::make_shared<CameraCalibration>(), rcal = std::make_shared<CameraCalibration>();
    lcal->setK(K[0], K[1], K[2], K[3]);
    rcal->setK(Kr[0], Kr[1], Kr[2], Kr[3]);
    // Trl = right-from-left; the reference stores Tc0ci (left-from-right) and inverts it (optimizer.cpp:112-114)
    rcal->Tc0ci_ = Sophus::SE3d(Eigen::Quaterniond(Trl[6], Trl[3], Trl[4], Trl[5]), Eigen::Vector3d(Trl[0], Trl[1], Trl[2])).inverse();
    for (int c = 0; c < ncam; ++c) {
        auto kf = std::make_shared<Frame>();
        kf->id_ = kf->kfid_ = c;
        kf->pcalib_leftcam_ = lcal; kf->pcalib_rightcam_ = rcal;
        const double* p = &pose[7 * c];
        kf->setTwc(Sophus::SE3d(Eigen::Quaterniond(p[6], p[3], p[4], p[5]), Eigen::Vector3d(p[0], p[1], p[2])));
        map->map_pkfs_[c] = kf;
    }
    for (int l = 0; l < npts; ++l) {
        auto lm = std::make_shared<MapPoint>();
        lm->lmid_ = l; lm->kfid_ = lac[l];
        auto kfa = map->map_pkfs_[lac[l]];
        const double z = 1.0 / invd[l];
        lm->ptxyz_ = kfa->getTwc() * (z * lcal->iK_ * Eigen::Vector3d((float)apx[2 * l], (float)apx[2 * l + 1], 1.0));
        lm->invdepth_ = invd[l];
        lm->set_kfids_.insert(lac[l]);
        Keypoint kp; kp.lmid_ = l; kp.is3d_ = true;
        kp.unpx_ = cv::Point2f((float)apx[2 * l], (float)apx[2 * l + 1]);
        kfa->mapkps_[l] = kp;
        map->map_plms_[l] = lm;
    }
    for (int i = 0; i < nobs; ++i) {
        auto kf = map->map_pkfs_[oc[i]];
        Keypoint& kp = kf->mapkps_[ol[i]];
        kp.lmid_ = ol[i]; kp.is3d_ = true;
        const cv::Point2f px((float)opx[2 * i], (float)opx[2 * i + 1]);
        if (oty[i] == 0) kp.unpx_ = px;
        else { kp.runpx_ = px; kp.is_stereo_ = true; }               // 1: other keyframe, 2: the anchor keyframe's own right view
        map->map_plms_[ol[i]]->set_kfids_.insert(oc[i]);
    }
    for (auto& kv : map->map_pkfs_) {
        kv.second->nbkps_ = kv.second->mapkps_.size();
        kv.second->nb3dkps_ = kv.second->mapkps_.size();
    }
    // the newest keyframe is the one localBA is called for; constant keyframes get a covisibility score below
    // nmin_covscore so that the window walk freezes them (optimizer.cpp:150-188)
    std::vector<Sophus::SE3d> anchors_before;
    for (int c = 0; c < ncam; ++c) anchors_before.push_back(map->map_pkfs_[c]->getTwc());
    auto newkf = map->map_pkfs_[ncam - 1];
    const std::string mode0 = argc > 3 ? argv[3] : "";
    // "gauge": every keyframe strongly covisible, none pre-marked constant - the gauge rule alone decides what is fixed
    for (int c = 0; c < ncam - 1; ++c) newkf->covkfs_[c] = (pc[c] && mode0 != "gauge") ? 0 : 1000;
    map->pcurframe_ = newkf;
    map->nkfid_ = ncam - 1;
    Optimizer opt(params, map);
    const std::string mode = argc > 3 ? argv[3] : "";
    Sophus::SE3d cur_before, new_before;
    if (mode == "loose" || mode == "full") {
        // the current frame is its own object in the reference (the map stores keyframe COPIES): looseBA moves it rigidly
        // with the loop keyframe (optimizer.cpp:1649-1653)
        auto cur = std::make_shared<Frame>(*newkf);
        cur->setTwc(newkf->getTwc() * Sophus::SE3d(Eigen::Quaterniond(1, 0, 0, 0), Eigen::Vector3d(0.1, -0.05, 0.2)));
        map->pcurframe_ = cur;
        cur_before = cur->getTwc();
        new_before = newkf->getTwc();
        if (mode == "loose") opt.looseBA(0, ncam - 1, true);
        else opt.fullBA(true);
    } else {
        if (mode == "stop") opt.signalStopLocalBA();
        opt.localBA(*newkf, true);
        if (opt.stopLocalBA()) { fprintf(stderr, "bstop_localba_ not cleared\n"); return 4; }
    }
    f = fopen(argv[2], "wb");
    if (!f) return 3;
    for (int c = 0; c < ncam; ++c) {
        const Sophus::SE3d T = map->map_pkfs_[c]->getTwc();
        const double p[7] = {T.translation().x(), T.translation().y(), T.translation().z(), T.unit_quaternion().x(),
                             T.unit_quaternion().y(), T.unit_quaternion().z(), T.unit_quaternion().w()};
        fwrite(p, sizeof(double), 7, f);
    }
    for (int l = 0; l < npts; ++l) {
        auto lm = map->getMapPoint(l);
        double v = lm ? lm->invdepth_ : -1.0;
        // looseBA updates the world point only (updateMapPoint(lmid, wpt), optimizer.cpp:1531-1535): report the inverse depth the
        // point has in its anchor keyframe AS THE SOLVE LEFT IT - looseBA forms the point with the anchor's pose before the
        // keyframes move, so the pre-solve pose is the one to look through (saved in anchors_before)
        if (lm && mode == "loose") v = 1.0 / (anchors_before[lac[l]].inverse() * lm->getPoint()).z();
        fwrite(&v, sizeof(double), 1, f);
    }
    if (mode == "loose") {
        // rigid follow-up of the current frame: Twcur' = Twnew_opt * (Tnew_w_ini * Twcur)
        const Sophus::SE3d expect = newkf->getTwc() * (new_before.inverse() * cur_before);
        const Sophus::SE3d got = map->pcurframe_->getTwc();
        const Eigen::Vector3d d = got.translation() - expect.translation();
        if (d.x() * d.x() + d.y() * d.y() + d.z() * d.z() > 1e-18) { fprintf(stderr, "current frame not moved with the loop keyframe\n"); return 5; }
    }
    const int32_t nrem = (int32_t)map->removed_obs_.size();
    fwrite(&nrem, 4, 1, f);
    fclose(f);
    printf("BA shim done: %d keyframes, %d map points, %d observations removed, %zu points removed\n", ncam, npts, nrem, map->removed_points_.size());
    return 0;
}
