// Mapper::matchToMap on the GPU (8f-4): the reference's declaration (include/mapper.hpp:92) is kept, this translation unit
// supplies the body: it FLATTENS what the two loops of /root/reference/src/mapper.cpp:576-774 read - the frame's pose,
// calibration, grid and keypoints; the candidate map points and the map points of the frame's keypoints with their
// descriptors, keyframe-observation sets and per-keyframe pixels; the observing keyframes' poses - makes ONE call of
// ov2_match_to_map (projection, culling, neighbourhood search, the three geometric / co-visibility tests, descriptor
// distances, best / second + ratio, per-keypoint winner: csrc/match_map.cu) and turns the answer back into the
// map<kp lmid, map-point lmid> the caller merges (mapper.cpp:559-570).  Exclude the reference's own body with
// #ifndef OV2_EXTERNAL_MATCHTOMAP.  Compile-checked and self-tested against the stand-in map classes (host/standin/ref/).
//
// Kept exactly: the candidate filter (:603-616), the iteration order of `set_local_lmids` (the same unordered_set, so the same
// order the reference would walk - it decides ties), the grid cells' list order, the map clean-up side effects
// (removeMapPointObs for observations whose keyframe or keypoint is gone, :670-672, :697-703 - done while flattening, i.e. for
// every keypoint of the frame rather than only for those the loop would have reached), dmaxpxdist doubling (:597-600).
// Not handled here: fisheye calibrations and more than 256 keyframes in the observation sets (diagnostic, empty result: use
// the reference's body for those), the early exit when a new keyframe arrives mid-loop (checked once, before the call).
#include <cmath>
#include <iostream>
#include <map>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "mapper.hpp"             // the reference's, unchanged
#include "abi_flat.hpp"
#include "../../include/ov2b200.h"

namespace {
ov2_ctx* match_context() {
    static ov2_ctx* ctx = nullptr;                    // mapper thread only
    if (!ctx && ov2_create(0, &ctx) != OV2_OK) ctx = nullptr;
    return ctx;
}
}  // namespace

std::map<int,int> Mapper::matchToMap(const Frame &frame, const float fmaxprojerr, const float fdistratio, std::unordered_set<int> &set_local_lmids)
{
    std::map<int,int> map_previd_newid;
    if (set_local_lmids.empty() || bnewkfavailable_) return map_previd_newid;             // :581-583, :605-607
    ov2_ctx* ctx = match_context();
    if (!ctx) { std::cerr << "[ov2b200] matchToMap: no CUDA device (no CPU fallback)\n"; return map_previd_newid; }
    auto cal = frame.pcalib_leftcam_;
    if (cal->model_ != CameraCalibration::Pinhole) {
        std::cerr << "[ov2b200] matchToMap: only the pinhole (radial-tangential) model is built; keep the reference's body for fisheye\n";
        return map_previd_newid;
    }
    // ---- field of view and radius (:585-600)
    const float vfov = 0.5 * cal->img_h_ / cal->fy_;
    const float hfov = 0.5 * cal->img_w_ / cal->fx_;
    const float maxradfov = hfov > vfov ? std::atan(hfov) : std::atan(vfov);
    const float view_th = std::cos(maxradfov);
    float dmaxpxdist = fmaxprojerr;
    if (frame.nb3dkps_ < 30) dmaxpxdist *= 2.;

    // ---- map-point table: index of a map-point id, created on first use
    std::unordered_map<int, int> mp_index;
    std::vector<std::shared_ptr<MapPoint>> mps;
    auto mp_of = [&](int lmid, const std::shared_ptr<MapPoint>& plm) {
        auto it = mp_index.find(lmid);
        if (it != mp_index.end()) return it->second;
        const int k = (int)mps.size();
        mp_index.emplace(lmid, k);
        mps.push_back(plm);
        return k;
    };
    // ---- candidates, in the set's own iteration order (:603-616)
    std::vector<int32_t> cand_mp;
    std::vector<int> cand_lmid;
    for (const int lmid : set_local_lmids) {
        if (frame.isObservingKp(lmid)) continue;
        auto plm = pmap_->getMapPoint(lmid);
        if (plm == nullptr) continue;
        if (!plm->is3d_ || plm->desc_.empty()) continue;
        cand_mp.push_back(mp_of(lmid, plm));
        cand_lmid.push_back(lmid);
    }
    // ---- the frame's keypoints and grid (Frame::getSurroundingKeypoints reads vgridkps_ + mapkps_, frame.cpp:624-650)
    const std::vector<Keypoint> vkps = frame.getKeypoints();
    std::vector<float> kp_px;
    std::vector<int32_t> kp_lm(vkps.size(), -1);
    for (size_t j = 0; j < vkps.size(); ++j) {
        const Keypoint& kp = vkps[j];
        kp_px.push_back(kp.px_.x);
        kp_px.push_back(kp.px_.y);
        if (kp.lmid_ < 0) continue;                                                        // :651-653
        auto pkplm = pmap_->getMapPoint(kp.lmid_);
        if (pkplm == nullptr) { pmap_->removeMapPointObs(kp.lmid_, frame.kfid_); continue; }   // :667-672
        if (pkplm->desc_.empty()) continue;                                                // :674-676
        kp_lm[j] = mp_of(kp.lmid_, pkplm);
    }
    std::vector<int32_t> cell_ptr, cell_kp;
    if (!ov2shim::grid_csr(frame, vkps, "matchToMap", cell_ptr, cell_kp)) return map_previd_newid;
    // ---- per map point: world point, descriptors, keyframe set (as raw as getKfObsSet() returns it), valid observations
    std::unordered_map<int, int> kf_index;
    std::vector<std::shared_ptr<Frame>> kfs;
    std::vector<double> mp_xyz, kf_Tcw;
    std::vector<int32_t> desc_ptr(1, 0), obs_ptr(1, 0), obs_kf;
    std::vector<uint8_t> desc;
    std::vector<uint64_t> kfmask(4 * mps.size(), 0);
    std::vector<float> obs_px;
    bool too_many_kfs = false;
    auto kf_of = [&](int kfid) {
        auto it = kf_index.find(kfid);
        if (it != kf_index.end()) return it->second;
        const int k = (int)kf_index.size();
        kf_index.emplace(kfid, k);
        kfs.push_back(pmap_->getKeyframe(kfid));
        return k;
    };
    // the keypoints' map points need their observation lists (co-projection test); the candidates only their keyframe sets
    std::vector<char> is_kp_mp(mps.size(), 0);
    for (const int32_t m : kp_lm) if (m >= 0) is_kp_mp[m] = 1;
    for (size_t m = 0; m < mps.size(); ++m) {
        const auto& plm = mps[m];
        const Eigen::Vector3d w = plm->getPoint();
        mp_xyz.push_back(w.x()); mp_xyz.push_back(w.y()); mp_xyz.push_back(w.z());
        for (const auto& kd : plm->map_kf_desc_) {
            if (kd.second.empty() || kd.second.cols < 32) continue;
            const unsigned char* p = kd.second.ptr(0);
            desc.insert(desc.end(), p, p + 32);
        }
        desc_ptr.push_back((int32_t)(desc.size() / 32));
        const int lmid = plm->lmid_;
        for (const int kfid : plm->getKfObsSet()) {
            const int k = kf_of(kfid);
            if (k >= 256) { too_many_kfs = true; continue; }
            kfmask[4 * m + (k >> 6)] |= (uint64_t)1 << (k & 63);
            if (!is_kp_mp[m]) continue;
            auto pcokf = kfs[k];
            if (pcokf == nullptr) { pmap_->removeMapPointObs(lmid, kfid); continue; }       // :700-703
            const Keypoint cokp = pcokf->getKeypointById(lmid);
            if (cokp.lmid_ != lmid) { pmap_->removeMapPointObs(lmid, kfid); continue; }     // :696-698
            obs_kf.push_back(k);
            obs_px.push_back(cokp.px_.x);
            obs_px.push_back(cokp.px_.y);
        }
        obs_ptr.push_back((int32_t)obs_kf.size());
    }
    if (too_many_kfs) {
        std::cerr << "[ov2b200] matchToMap: more than 256 keyframes in the observation sets; keep the reference's body for maps this large\n";
        return map_previd_newid;
    }
    kf_Tcw.assign(12 * kfs.size(), 0.0);
    for (size_t k = 0; k < kfs.size(); ++k)
        if (kfs[k]) ov2shim::put_pose(kfs[k]->getTcw(), &kf_Tcw[12 * k]);
    // ---- one call
    ov2_match_problem p{};
    ov2shim::put_pose(frame.getTcw(), p.Tcw);
    double D[5];
    p.dist = ov2shim::put_pinhole(*cal, p.K, D);
    p.img_w = (int)cal->img_w_; p.img_h = (int)cal->img_h_;
    p.ncellsize = (int)frame.ncellsize_; p.nbwcells = (int)frame.nbwcells_; p.ncells = (int)frame.vgridkps_.size();
    p.cell_ptr = cell_ptr.data(); p.cell_kp = cell_kp.data();
    p.nkps = (int)vkps.size(); p.kp_px = kp_px.data(); p.kp_lm = kp_lm.data();
    p.nmps = (int)mps.size(); p.mp_xyz = mp_xyz.data(); p.mp_desc_ptr = desc_ptr.data(); p.ndesc = (int)(desc.size() / 32); p.desc = desc.data();
    p.mp_kfmask = kfmask.data(); p.mp_obs_ptr = obs_ptr.data(); p.nobs = (int)obs_kf.size(); p.obs_kf = obs_kf.data(); p.obs_px = obs_px.data();
    p.nkfs = (int)kfs.size(); p.kf_Tcw = kf_Tcw.data();
    p.ncand = (int)cand_mp.size(); p.cand_mp = cand_mp.data();
    p.dmaxpxdist = dmaxpxdist; p.fdistratio = fdistratio; p.view_th = view_th;
    if (p.ncand == 0 || p.nkps == 0) return map_previd_newid;
    std::vector<int32_t> best_kp(p.ncand), kp_match(p.nkps);
    std::vector<float> best_dist(p.ncand), kp_dist(p.nkps);
    if (ov2_match_to_map(ctx, &p, best_kp.data(), best_dist.data(), kp_match.data(), kp_dist.data()) != OV2_OK) {
        std::cerr << "[ov2b200] matchToMap: " << ov2_last_error(ctx) << "\n";
        return map_previd_newid;
    }
    for (size_t j = 0; j < vkps.size(); ++j)
        if (kp_match[j] >= 0) map_previd_newid.emplace(vkps[j].lmid_, cand_lmid[kp_match[j]]);   // :766-768
    return map_previd_newid;
}
