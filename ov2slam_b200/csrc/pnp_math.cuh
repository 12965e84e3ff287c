// MultiViewGeometry::ceresPnP ("next" row 2, SURVEY.md 8f; /root/reference/src/multi_view_geometry.cpp:492-588):
// motion-only bundle adjustment of ONE pose against N fixed 3D points, ReprojectionErrorSE3 residuals
// (src/ceres_parametrization.cpp:300-356), Huber loss, Ceres 2.0 trust-region loop with the
// Levenberg-Marquardt strategy, two-stage outlier flow.  Restated in oracle/pnp_ref.py.
//
// The whole solve is ONE function template over a parallel context `Par`:
//   begin() / stride()   which points this execution lane owns,
//   reduce(v, n)         all-reduce (sum) of n <= 32 doubles, the same bits returned to every lane,
//   sync()               barrier.
// On the GPU (pnp_solver.cu) Par is a thread block: every thread runs the controller redundantly on
// block-reduced sums, so the control flow is uniform.  On the host (tests/test_host_logic.py) Par is a
// single lane: the SAME code is compiled with g++ and compared with the oracle.
//
// Linear algebra: the reference asks Ceres for DENSE_QR on [J; sqrt(D)]; here the 6 x 6 damped normal
// equations are formed by the reduction and solved by LDL' in double.  Same minimiser; the difference
// is rounding (cond(J)^2 ~ 1e6 at PnP geometry), inside the 1e-9 pose tolerance of the tests (the kernel on an H100 lands
// within 1.2e-13 of the oracle on tests/test_pnp_paths_gpu.py, n = 1 and 2 and KITTI-scale poses included).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PNP_HD __host__ __device__ inline
#else
#define PNP_HD inline
#endif

namespace pnp {

constexpr double SOPHUS_EPS = 1e-10;
constexpr double DBLMAX = 1.7976931348623157e308;

PNP_HD void quat_to_rot(const double* q, double* R) {   // unit quaternion [x y z w] -> row-major R (Eigen toRotationMatrix)
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// SE3LeftParameterization::Plus: out = Sophus::SE3d::exp(d) * (q, t); pose = [t(3), q(xyzw)]
PNP_HD void pose_plus(const double* pose, const double* d, double* out) {
    double q[4] = {pose[3], pose[4], pose[5], pose[6]};
    const double qn = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) q[i] *= qn;
    const double ox = d[3], oy = d[4], oz = d[5];
    const double th2 = ox * ox + oy * oy + oz * oz;
    double imag, real, theta;
    if (th2 < SOPHUS_EPS * SOPHUS_EPS) {
        theta = 0.0;
        const double th4 = th2 * th2;
        imag = 0.5 - (1.0 / 48.0) * th2 + (1.0 / 3840.0) * th4;
        real = 1.0 - (1.0 / 8.0) * th2 + (1.0 / 384.0) * th4;
    } else {
        theta = sqrt(th2);
        imag = sin(0.5 * theta) / theta;
        real = cos(0.5 * theta);
    }
    const double e[4] = {imag * ox, imag * oy, imag * oz, real};
    double Re[9], V[9];
    quat_to_rot(e, Re);
    if (theta < SOPHUS_EPS) {
        for (int i = 0; i < 9; ++i) V[i] = Re[i];
    } else {
        const double a = (1.0 - cos(theta)) / th2;
        const double b = (theta - sin(theta)) / (th2 * theta);
        const double O[9] = {0, -oz, oy, oz, 0, -ox, -oy, ox, 0};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                const double o2 = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
                V[3 * i + j] = a * O[3 * i + j] + b * o2 + (i == j ? 1.0 : 0.0);
            }
    }
    const double* t = pose;
    double r[4];
    r[3] = e[3] * q[3] - e[0] * q[0] - e[1] * q[1] - e[2] * q[2];
    r[0] = e[3] * q[0] + e[0] * q[3] + e[1] * q[2] - e[2] * q[1];
    r[1] = e[3] * q[1] + e[1] * q[3] + e[2] * q[0] - e[0] * q[2];
    r[2] = e[3] * q[2] + e[2] * q[3] + e[0] * q[1] - e[1] * q[0];
    const double n = 1.0 / sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
    for (int i = 0; i < 3; ++i)
        out[i] = V[3 * i] * d[0] + V[3 * i + 1] * d[1] + V[3 * i + 2] * d[2] + Re[3 * i] * t[0] + Re[3 * i + 1] * t[1] + Re[3 * i + 2] * t[2];
    out[3] = r[0] * n; out[4] = r[1] * n; out[5] = r[2] * n; out[6] = r[3] * n;
}

struct Problem {
    int n;
    const double* unpx;      // [n][2]
    const double* wpts;      // [n][3]
    const int32_t* scales;   // [n] or NULL: residuals scaled by 2^-scale
    double K[4];             // fx fy cx cy
};

struct Summary {
    int iterations;
    int termination;         // 0 convergence, 1 no convergence (iteration cap), 2 failure
    double initial_cost, final_cost;
};

// One Evaluate() of every active block at `pose`.  acc (28) += [H upper triangle (21) | g (6) | cost] of the
// loss-corrected Gauss-Newton model when jac, [.. | cost] otherwise; chi2 / depth flags of the blocks are stored.
template <class Par>
PNP_HD void evaluate(Par& par, const Problem& P, const uint8_t* active, const double* pose, double huber_a, bool jac,
                     double* acc, double* last_chi2, uint8_t* last_depth) {
    double q[4] = {pose[3], pose[4], pose[5], pose[6]};
    const double qn = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) q[i] *= qn;
    double Rwc[9];
    quat_to_rot(q, Rwc);
    const double fx = P.K[0], fy = P.K[1], cx = P.K[2], cy = P.K[3];
    for (int i = 0; i < 28; ++i) acc[i] = 0.0;
    for (int p = par.begin(); p < P.n; p += par.stride()) {
        if (active && !active[p]) continue;
        const double* w = P.wpts + 3 * (size_t)p;
        const double dx = w[0] - pose[0], dy = w[1] - pose[1], dz = w[2] - pose[2];
        // Tcw * wpt = Rwc' (wpt - twc)
        const double X = Rwc[0] * dx + Rwc[3] * dy + Rwc[6] * dz;
        const double Y = Rwc[1] * dx + Rwc[4] * dy + Rwc[7] * dz;
        const double Z = Rwc[2] * dx + Rwc[5] * dy + Rwc[8] * dz;
        const double invz = 1.0 / Z;
        const double sinfo = P.scales ? 1.0 / pow(2.0, (double)P.scales[p]) : 1.0;
        const double r0 = (fx * X * invz + cx - P.unpx[2 * (size_t)p]) * sinfo;
        const double r1 = (fy * Y * invz + cy - P.unpx[2 * (size_t)p + 1]) * sinfo;
        const double s = r0 * r0 + r1 * r1;
        last_chi2[p] = s;
        last_depth[p] = Z > 0.0 ? 1 : 0;
        double rho0 = s, wgt = 1.0;                      // HuberLoss(a): rho, sqrt(rho') (rho'' <= 0: the corrector only rescales)
        if (huber_a > 0.0 && s > huber_a * huber_a) {
            const double rs = sqrt(s);
            rho0 = 2.0 * huber_a * rs - huber_a * huber_a;
            double rho1 = huber_a / rs;
            if (rho1 < 2.2250738585072014e-308) rho1 = 2.2250738585072014e-308;
            wgt = sqrt(rho1);
        }
        acc[27] += 0.5 * rho0;
        if (!jac) continue;
        const double invz2 = invz * invz;
        // J_cam (2x3) Rcw, Rcw = Rwc'
        const double a00 = invz * fx, a02 = -X * invz2 * fx, a11 = invz * fy, a12 = -Y * invz2 * fy;
        double JR[6];
        for (int j = 0; j < 3; ++j) {                    // Rcw(i, j) = Rwc[3 j + i]
            JR[j] = a00 * Rwc[3 * j] + a02 * Rwc[3 * j + 2];
            JR[3 + j] = a11 * Rwc[3 * j + 1] + a12 * Rwc[3 * j + 2];
        }
        double J[12];
        const double sw = sinfo * wgt;
        for (int i = 0; i < 2; ++i) {
            const double* jr = JR + 3 * i;
            J[6 * i + 0] = -jr[0] * sw;
            J[6 * i + 1] = -jr[1] * sw;
            J[6 * i + 2] = -jr[2] * sw;
            // JR * hat(wpt): hat(w) = [0 -w2 w1; w2 0 -w0; -w1 w0 0]
            J[6 * i + 3] = (jr[1] * w[2] - jr[2] * w[1]) * sw;
            J[6 * i + 4] = (jr[2] * w[0] - jr[0] * w[2]) * sw;
            J[6 * i + 5] = (jr[0] * w[1] - jr[1] * w[0]) * sw;
        }
        const double e0 = r0 * wgt, e1 = r1 * wgt;
        int k = 0;
        for (int a = 0; a < 6; ++a) {
            for (int b = a; b < 6; ++b) acc[k++] += J[a] * J[b] + J[6 + a] * J[6 + b];
            acc[21 + a] += J[a] * e0 + J[6 + a] * e1;
        }
    }
    par.reduce(acc, 28);
}

// (H + diag(d2)) x = -g by LDL' (6 x 6, H given as the upper triangle in row order); false if not positive definite
PNP_HD bool solve6(const double* Hup, const double* d2, const double* g, double* x) {
    double A[36];
    int k = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) { A[6 * a + b] = Hup[k]; A[6 * b + a] = Hup[k]; ++k; }
    for (int a = 0; a < 6; ++a) A[7 * a] += d2[a];
    double L[36], D[6];
    for (int j = 0; j < 6; ++j) {
        double dj = A[7 * j];
        for (int m = 0; m < j; ++m) dj -= L[6 * j + m] * L[6 * j + m] * D[m];
        if (!(dj > 0.0) || !isfinite(dj)) return false;
        D[j] = dj;
        for (int i = j + 1; i < 6; ++i) {
            double v = A[6 * i + j];
            for (int m = 0; m < j; ++m) v -= L[6 * i + m] * L[6 * j + m] * D[m];
            L[6 * i + j] = v / dj;
        }
    }
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double v = -g[i];
        for (int m = 0; m < i; ++m) v -= L[6 * i + m] * y[m];
        y[i] = v;
    }
    for (int i = 5; i >= 0; --i) {
        double v = y[i] / D[i];
        for (int m = i + 1; m < 6; ++m) v -= L[6 * m + i] * x[m];
        x[i] = v;
    }
    return true;
}

// ceres::Solve on the active blocks (trust_region_minimizer.cc flow as restated in oracle/pnp_ref.py::ceres_solve_pose)
template <class Par>
PNP_HD void solve_pose(Par& par, const Problem& P, const uint8_t* active, double* pose, int max_iters, double huber_a,
                       double function_tolerance, double* last_chi2, uint8_t* last_depth, Summary& S) {
    double acc[28], x[7], best[7];
    {
        const double zero[6] = {0, 0, 0, 0, 0, 0};
        pose_plus(pose, zero, x);                           // normalises the quaternion like SE3d(q, t)
        x[0] = pose[0]; x[1] = pose[1]; x[2] = pose[2];
    }
    for (int i = 0; i < 7; ++i) best[i] = x[i];
    evaluate(par, P, active, x, huber_a, true, acc, last_chi2, last_depth);
    double x_cost = acc[27];
    double scale[6], Hs[21], gs[6];
    {
        int k = 0;
        for (int a = 0; a < 6; ++a) { scale[a] = 1.0 / (1.0 + sqrt(acc[k])); k += 6 - a; }   // jacobi scaling, once
    }
    auto rescale = [&](const double* a_) {
        int k = 0;
        for (int a = 0; a < 6; ++a) {
            for (int b = a; b < 6; ++b) { Hs[k] = a_[k] * scale[a] * scale[b]; ++k; }
            gs[a] = a_[21 + a] * scale[a];
        }
    };
    auto grad_max = [&](const double* xx, const double* a_) {
        double mg[6], xp[7], m = 0.0;
        for (int a = 0; a < 6; ++a) mg[a] = -a_[21 + a];
        pose_plus(xx, mg, xp);
        for (int i = 0; i < 7; ++i) m = fmax(m, fabs(xx[i] - xp[i]));
        return m;
    };
    double gmax = grad_max(x, acc);
    rescale(acc);
    S.initial_cost = x_cost;
    S.termination = 1;
    double minimum_cost = DBLMAX, xnorm = -1.0, radius = 1e4, decrease = 2.0, diag[6];
    bool reuse_diag = false, step_ok = true;
    int num_invalid = 0, it = 0;
    for (;;) {
        if (step_ok && x_cost < minimum_cost) {
            minimum_cost = x_cost;
            for (int i = 0; i < 7; ++i) best[i] = x[i];
        }
        if (it >= max_iters) break;
        if (step_ok && gmax <= 1e-10) { S.termination = 0; break; }
        if (radius <= 1e-32) { S.termination = 0; break; }
        ++it;
        if (!reuse_diag) {
            int k = 0;
            for (int a = 0; a < 6; ++a) { diag[a] = fmin(fmax(Hs[k], 1e-6), 1e32); k += 6 - a; }
        }
        reuse_diag = true;
        double d2[6], step[6];
        for (int a = 0; a < 6; ++a) d2[a] = diag[a] / radius;
        bool valid = solve6(Hs, d2, gs, step);
        double mcc = 0.0;
        if (valid) {
            // model cost change -(J s)'(r + J s / 2) = -(s'g + s'H s / 2)
            double sg = 0.0, sHs = 0.0;
            int k = 0;
            for (int a = 0; a < 6; ++a) {
                sg += step[a] * gs[a];
                for (int b = a; b < 6; ++b) { sHs += (a == b ? 1.0 : 2.0) * step[a] * step[b] * Hs[k]; ++k; }
            }
            mcc = -(sg + 0.5 * sHs);
            for (int a = 0; a < 6; ++a) valid = valid && isfinite(step[a]);
            valid = valid && mcc > 0.0;
        }
        if (!valid) {
            if (++num_invalid >= 5) { S.termination = 2; break; }
            radius /= decrease; decrease *= 2.0;
            step_ok = false;
            continue;
        }
        num_invalid = 0;
        double delta[6], cand[7];
        for (int a = 0; a < 6; ++a) delta[a] = step[a] * scale[a];
        pose_plus(x, delta, cand);
        evaluate(par, P, active, cand, huber_a, false, acc, last_chi2, last_depth);
        double cand_cost = acc[27];
        if (!isfinite(cand_cost)) cand_cost = DBLMAX;
        double sn = 0.0;
        for (int i = 0; i < 7; ++i) sn += (x[i] - cand[i]) * (x[i] - cand[i]);
        if (sqrt(sn) <= 1e-8 * (xnorm + 1e-8)) { S.termination = 0; break; }
        if (fabs(x_cost - cand_cost) <= function_tolerance * x_cost) { S.termination = 0; break; }
        const double rel = cand_cost >= DBLMAX ? -DBLMAX : (x_cost - cand_cost) / mcc;
        if (rel > 1e-3) {
            for (int i = 0; i < 7; ++i) x[i] = cand[i];
            double xn = 0.0;
            for (int i = 0; i < 7; ++i) xn += x[i] * x[i];
            xnorm = sqrt(xn);
            evaluate(par, P, active, x, huber_a, true, acc, last_chi2, last_depth);
            x_cost = acc[27];
            gmax = grad_max(x, acc);
            rescale(acc);
            step_ok = true;
            const double t = 2.0 * rel - 1.0;
            radius = fmin(1e16, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
            decrease = 2.0;
            reuse_diag = false;
        } else {
            step_ok = false;
            radius /= decrease; decrease *= 2.0;
        }
    }
    S.iterations = it;
    S.final_cost = minimum_cost < DBLMAX ? minimum_cost : x_cost;
    for (int i = 0; i < 7; ++i) pose[i] = best[i];
}

// MultiViewGeometry::ceresPnP.  `flags` [n] receives 1 for the blocks the scan after the first solve rejects
// (chi2 > chi2th or depth <= 0); `work` [n] is scratch for the second solve's active mask.  Returns success.
template <class Par>
PNP_HD bool ceres_pnp(Par& par, const Problem& P, double* pose, int nmaxiter, float chi2th, bool use_robust, bool apply_l2,
                      double* last_chi2, uint8_t* last_depth, uint8_t* flags, uint8_t* work, Summary& S) {
    double p[7];
    for (int i = 0; i < 7; ++i) p[i] = pose[i];
    const double a = use_robust ? (double)sqrtf(chi2th) : 0.0;
    solve_pose(par, P, nullptr, p, nmaxiter, a, 1e-3, last_chi2, last_depth, S);
    double nbad = 0.0;
    for (int i = par.begin(); i < P.n; i += par.stride()) {
        const bool bad = last_chi2[i] > (double)chi2th || !last_depth[i];
        flags[i] = bad ? 1 : 0;
        work[i] = bad ? 0 : 1;
        nbad += bad ? 1.0 : 0.0;
    }
    par.reduce(&nbad, 1);
    par.sync();
    if ((int)nbad == P.n) return false;                  // Twc is not written back (multi_view_geometry.cpp:568-570)
    if (apply_l2 && nbad > 0.0) solve_pose(par, P, work, p, nmaxiter, 0.0, 1e-3, last_chi2, last_depth, S);
    for (int i = 0; i < 7; ++i) pose[i] = p[i];
    return S.termination != 2;                           // Summary::IsSolutionUsable()
}

struct SerialPar {                                       // host / single-lane context
    PNP_HD int begin() const { return 0; }
    PNP_HD int stride() const { return 1; }
    PNP_HD void reduce(double*, int) {}
    PNP_HD void sync() {}
};

}  // namespace pnp
