// MultiViewGeometry::ceresPnP on the GPU: link-time replacement of the two static overloads
// (/root/reference/include/multi_view_geometry.hpp:82-93; bodies src/multi_view_geometry.cpp:492-588), which
// VisualFrontEnd::computePose calls every frame right after tracking (src/visual_front_end.cpp:791-801).  The rest of
// MultiViewGeometry (P3P / 5-point RANSAC, triangulation) stays in the reference's own translation unit built with
// -DOV2_EXTERNAL_CERESPNP (one #ifndef around the two bodies, INTEGRATION.md).
//
// Same arguments, same return value (false when every block was rejected, Twc untouched then, or when the solve was not
// usable; false for an empty input), voutliersidx filled with the rejected residual blocks.  voutliersidx is cleared first,
// where the reference appends to it: both callers pass an empty vector, so the results are the same.  The 5 ms wall-clock cap of the reference (:545-546) is not
// modelled (the device solve takes tens of microseconds).  No CPU fallback: without a device the call reports and
// returns false (the caller then keeps the P3P / motion-model pose, exactly as after a failed Ceres solve).
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "multi_view_geometry.hpp"
#include "../../include/ov2b200.h"

namespace {
struct PnpState { ov2_ctx* ctx = nullptr; std::mutex mu; bool failed = false; };
PnpState& pnp_state() { static PnpState s; return s; }
}  // namespace

bool MultiViewGeometry::ceresPnP(const std::vector<Eigen::Vector2d, Eigen::aligned_allocator<Eigen::Vector2d> > &vunkps,
                                 const std::vector<Eigen::Vector3d, Eigen::aligned_allocator<Eigen::Vector3d> > &vwpts,
                                 Sophus::SE3d &Twc, const int nmaxiter, const float chi2th, const bool buse_robust,
                                 const bool bapply_l2_after_robust, const float fx, const float fy, const float cx, const float cy,
                                 std::vector<int> &voutliersidx)
{
    // multi_view_geometry.cpp:492-505: the scale-less overload is the scaled one with every keypoint at level 0
    std::vector<int> vscales(vunkps.size(), 0);
    return ceresPnP(vunkps, vwpts, vscales, Twc, nmaxiter, chi2th, buse_robust, bapply_l2_after_robust, fx, fy, cx, cy, voutliersidx);
}

bool MultiViewGeometry::ceresPnP(const std::vector<Eigen::Vector2d, Eigen::aligned_allocator<Eigen::Vector2d> > &vunkps,
                                 const std::vector<Eigen::Vector3d, Eigen::aligned_allocator<Eigen::Vector3d> > &vwpts,
                                 const std::vector<int> &vscales, Sophus::SE3d &Twc, const int nmaxiter, const float chi2th,
                                 const bool buse_robust, const bool bapply_l2_after_robust, const float fx, const float fy,
                                 const float cx, const float cy, std::vector<int> &voutliersidx)
{
    const size_t n = vunkps.size();
    if (n == 0 || vwpts.size() != n || vscales.size() != n) return false;            // (:507-509 asserts equal sizes)
    PnpState& s = pnp_state();
    std::lock_guard<std::mutex> lk(s.mu);
    if (!s.ctx && !s.failed) {
        // the reference's class takes no device: OV2_DEVICE names the GPU (default 0)
        const char* e = getenv("OV2_DEVICE");
        if (ov2_create(e ? atoi(e) : 0, &s.ctx) != OV2_OK) {
            fprintf(stderr, "[ov2b200] ceresPnP: no CUDA device - the GPU path has no CPU fallback\n");
            s.ctx = nullptr; s.failed = true;
        }
    }
    if (!s.ctx) return false;
    std::vector<double> px(2 * n), wp(3 * n);
    std::vector<int32_t> sc(n);
    for (size_t i = 0; i < n; ++i) {
        px[2 * i] = vunkps[i].x(); px[2 * i + 1] = vunkps[i].y();
        wp[3 * i] = vwpts[i].x(); wp[3 * i + 1] = vwpts[i].y(); wp[3 * i + 2] = vwpts[i].z();
        sc[i] = vscales[i];
    }
    const int32_t off[2] = {0, (int32_t)n};
    const double K[4] = {fx, fy, cx, cy};
    const Eigen::Quaterniond q = Twc.unit_quaternion();
    const Eigen::Vector3d t = Twc.translation();
    double pose[7] = {t.x(), t.y(), t.z(), q.x(), q.y(), q.z(), q.w()};
    std::vector<uint8_t> flags(n, 0);
    uint8_t ok = 0;
    int32_t its = 0;
    if (ov2_pnp_solve(s.ctx, 1, off, px.data(), wp.data(), sc.data(), K, pose, nmaxiter, chi2th, buse_robust ? 1 : 0,
                      bapply_l2_after_robust ? 1 : 0, flags.data(), &ok, &its) != OV2_OK) {
        fprintf(stderr, "[ov2b200] ceresPnP: %s\n", ov2_last_error(s.ctx));
        return false;
    }
    voutliersidx.clear();
    for (size_t i = 0; i < n; ++i)
        if (flags[i]) voutliersidx.push_back((int)i);
    if (!ok) return false;                                                            // Twc untouched (:570-575)
    Twc = Sophus::SE3d(Eigen::Quaterniond(pose[6], pose[3], pose[4], pose[5]), Eigen::Vector3d(pose[0], pose[1], pose[2]));
    return true;
}
