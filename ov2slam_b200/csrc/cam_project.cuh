// Projection of a world point into a frame, shared by match_map.cu, frontend_klt_tracking.cu and frontend_stereo_matching.cu,
// and the undistortion of a pixel.
//
// Frame::projWorldToCam (src/frame.cpp:811-828) with the pose as 12 doubles (row-major rotation, then the translation), and
// CameraCalibration::projectCamToImageDist (src/camera_calibration.cpp:254-281) for the pinhole model, with or without
// radial-tangential distortion evaluated as cv::projectPoints does on the float-rounded normalised point.
// Files including this header are compiled with -fmad=false: every double is formed in the operation order written here,
// which oracle/match_ref.py (camera_point, project_dist) restates.
#pragma once

struct CamModel {
    double fx, fy, cx, cy, k1, k2, p1, p2, k3;
    int has_dist;
};

__host__ __device__ inline CamModel make_cam(const double* K, const double* dist) {
    CamModel c;
    c.fx = K[0]; c.fy = K[1]; c.cx = K[2]; c.cy = K[3];
    c.has_dist = dist ? 1 : 0;
    c.k1 = c.k2 = c.p1 = c.p2 = c.k3 = 0.0;
    if (dist) { c.k1 = dist[0]; c.k2 = dist[1]; c.p1 = dist[2]; c.p2 = dist[3]; c.k3 = dist[4]; }
    return c;
}

// camera-frame point T * w, each row summed left to right
__device__ __forceinline__ void transform(const double* T, const double* w, double& X, double& Y, double& Z) {
    X = T[0] * w[0] + T[1] * w[1] + T[2] * w[2] + T[9];
    Y = T[3] * w[0] + T[4] * w[1] + T[5] * w[2] + T[10];
    Z = T[6] * w[0] + T[7] * w[1] + T[8] * w[2] + T[11];
}

// CameraCalibration::projectCamToImageDist, pinhole model.  Z is not tested: a point behind the camera projects as the
// reference projects it.
__device__ __forceinline__ float2 project_dist(const CamModel& C, double X, double Y, double Z) {
    const double invz = 1.0 / Z;
    double x = X * invz, y = Y * invz;
    if (!C.has_dist) return make_float2((float)(C.fx * x + C.cx), (float)(C.fy * y + C.cy));
    x = (double)(float)x;                  // cv::Point3f(x, y, 1.)
    y = (double)(float)y;
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
    const double cdist = 1 + C.k1 * r2 + C.k2 * r4 + C.k3 * r6;
    const double xd = x * cdist + C.p1 * a1 + C.p2 * a2;
    const double yd = y * cdist + C.p1 * a3 + C.p2 * a1;
    return make_float2((float)(xd * C.fx + C.cx), (float)(yd * C.fy + C.cy));
}

// Frame::isInImage / isInRightImage (src/frame.cpp:840-848): float coordinates against the int image size
__device__ __forceinline__ bool in_image(float2 p, int img_w, int img_h) {
    return p.x >= 0.f && p.y >= 0.f && p.x < (float)img_w && p.y < (float)img_h;
}

// CameraCalibration::undistortImagePoint (src/camera_calibration.cpp:313-332), pinhole model: the pixel itself without
// distortion, else cv::undistortPoints(pt, K, D, K) as OpenCV evaluates it with its default criteria (5 iterations, no
// tolerance test) and D = (k1, k2, p1, p2, k3): the rational and thin-prism coefficients are zero, the tilt matrix and
// R are identities and P = K, so those terms add or multiply exact zeros and ones and are left out.  When the inverse
// radial factor turns negative the point keeps its normalised pixel coordinates (OpenCV's icdist < 0 exit).
// oracle/stereo_matching_ref.py::undistort_points_ref restates it; it equals cv2.undistortPoints bit for bit.
__host__ __device__ inline float2 undistort_point(const CamModel& C, float u, float v) {
    if (!C.has_dist) return make_float2(u, v);
    const double ifx = 1. / C.fx, ify = 1. / C.fy;
    const double x0 = ((double)u - C.cx) * ifx, y0 = ((double)v - C.cy) * ify;
    double x = x0, y = y0;
    for (int j = 0; j < 5; ++j) {
        const double r2 = x * x + y * y;
        const double icdist = 1. / (1 + ((C.k3 * r2 + C.k2) * r2 + C.k1) * r2);
        if (icdist < 0) {
            x = x0;
            y = y0;
            break;
        }
        const double dx = 2 * C.p1 * x * y + C.p2 * (r2 + 2 * x * x);
        const double dy = C.p1 * (r2 + 2 * y * y) + 2 * C.p2 * x * y;
        x = (x0 - dx) * icdist;
        y = (y0 - dy) * icdist;
    }
    return make_float2((float)(C.fx * x + C.cx), (float)(C.fy * y + C.cy));
}
