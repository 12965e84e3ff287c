// The reference's map objects as the flat arrays of the C ABI (include/ov2b200.h): the conversions the drop-ins that flatten a
// frame share (host/mapper_match_gpu.cpp, host/visual_front_end_klt_gpu.cpp, host/map_manager_stereo_gpu.cpp).  Matrices are read
// through their columns (M * e_j), so the same code compiles against Eigen and against the stand-in Eigen of host/standin/ref.
#pragma once
#include <cstdint>
#include <iostream>
#include <unordered_map>
#include <vector>

#include "frame.hpp"

namespace ov2shim {

// 9 doubles, row-major
inline void put_mat3(const Eigen::Matrix3d& M, double* out) {
    const Eigen::Vector3d c0 = M * Eigen::Vector3d(1, 0, 0), c1 = M * Eigen::Vector3d(0, 1, 0), c2 = M * Eigen::Vector3d(0, 0, 1);
    const double m[9] = {c0.x(), c1.x(), c2.x(), c0.y(), c1.y(), c2.y(), c0.z(), c1.z(), c2.z()};
    for (int i = 0; i < 9; ++i) out[i] = m[i];
}

// 12 doubles: the row-major rotation, then the translation
inline void put_pose(const Sophus::SE3d& T, double* out) {
    put_mat3(T.rotationMatrix(), out);
    const Eigen::Vector3d t = T.translation();
    out[9] = t.x(); out[10] = t.y(); out[11] = t.z();
}

// K = fx, fy, cx, cy and D = k1, k2, p1, p2, k3 of a pinhole (radial-tangential) calibration; CameraCalibration keeps four
// coefficients, so k3 = 0.  Returns D, or NULL when the calibration has no distortion model (Dcv_ empty,
// camera_calibration.cpp:262).
inline const double* put_pinhole(const CameraCalibration& cal, double* K, double* D) {
    K[0] = cal.fx_; K[1] = cal.fy_; K[2] = cal.cx_; K[3] = cal.cy_;
    D[0] = cal.k1_; D[1] = cal.k2_; D[2] = cal.p1_; D[3] = cal.p2_; D[4] = 0.0;
    return cal.Dcv_.empty() ? nullptr : D;
}

// Frame::vgridkps_ as a CSR of indices into `vkps` (cells row-major, each cell's ids in list order; ids that are not in vkps are
// skipped, as Frame::getSurroundingKeypoints skips them).  The ABI stages one grid entry per keypoint: a grid that lists fewer
// keypoints than vkps holds is padded with 0 (the padding is never reached through cell_ptr); one that lists more (an id in two
// cells) is not something the reference's Frame produces, and is refused with a diagnostic naming `who`.
inline bool grid_csr(const Frame& frame, const std::vector<Keypoint>& vkps, const char* who, std::vector<int32_t>& cell_ptr,
                     std::vector<int32_t>& cell_kps) {
    std::unordered_map<int, int32_t> index;
    for (size_t j = 0; j < vkps.size(); ++j) index.emplace(vkps[j].lmid_, (int32_t)j);
    const size_t ncells = frame.vgridkps_.size();
    cell_ptr.assign(ncells + 1, 0);
    cell_kps.clear();
    for (size_t c = 0; c < ncells; ++c) {
        for (const int id : frame.vgridkps_[c]) {
            auto it = index.find(id);
            if (it != index.end()) cell_kps.push_back(it->second);
        }
        cell_ptr[c + 1] = (int32_t)cell_kps.size();
    }
    if (cell_kps.size() > vkps.size()) {
        std::cerr << "[ov2b200] " << who << ": the frame's grid lists more keypoints than the frame holds\n";
        return false;
    }
    cell_kps.resize(vkps.size(), 0);
    return true;
}

}  // namespace ov2shim
