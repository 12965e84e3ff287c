// L: local bundle adjustment as ONE persistent kernel per solve (float64), device-side LM controller.
//
// Reference behaviour replaced: the solve sections of Optimizer::localBA
// (/root/reference/src/optimizer.cpp:436-479 robust solve, :492-594 outlier scan, :603-627 refinement,
// :637-735 second scan), i.e. Ceres 2.0's TrustRegionMinimizer (trust_region_minimizer.cc:67-134) +
// LevenbergMarquardtStrategy (levenberg_marquardt_strategy.cc:66-160) + Schur linear solver
// (schur_eliminator_impl.h:179-377) on the anchored inverse-depth residual blocks
// (src/ceres_parametrization.cpp:361-712) with SE3LeftParameterization (se3left_parametrization.hpp:41-60).
//
// Design: a solve is launch/sync-latency bound (C3: 0.66 MB per LM iteration, all of it L2 resident), so
// the whole two-stage solve - both Ceres solves, both outlier scans, every LM iteration - is ONE kernel
// launch.  A "group" of G CTAs works on one window; the phases of an LM iteration are separated by a group
// barrier (monotonic counter in global memory, release/acquire), not by kernel boundaries:
//
//   A  residual blocks + analytic Jacobians at x (thread per observation, keyframe rotations staged in the CTA's
//      keyframe table), cost                                                       [only when x changed]
//   B  Schur elimination, one warp per landmark, fp64 RED into the reduced camera system
//   B2 multi-GPU only: the partial systems of all ranks are summed straight out of peer memory over NVLink (no NCCL
//      call, no host round trip)
//   C  reduced camera system: LM damping + solve (n <= 96: Gauss-Jordan in CTA 0's shared memory; larger: blocked
//      Cholesky, sequential part on CTA 0, FP64 tensor-core trailing update spread over the group), gradient
//      projection by the last CTA
//   D  back-substitution + candidate point + candidate cost (warp per landmark; candidate poses are computed
//      redundantly by every CTA into shared memory)
//   E  the trust-region controller (ba_lm_ctl.cuh) replayed by every CTA from the same reduced scalars: all CTAs
//      take the same accept / reject / stop decision without a broadcast and without the host.
//
// K windows can be solved by one launch (ov2_localba_solve_batch): groups pull windows round-robin.
#include "ov2_common.cuh"
#include "ba_lm.cuh"
#include "ba_lm_ctl.cuh"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <mutex>
#include <thread>

namespace balm {

// ------------------------------------------------------------------ small SE3 helpers
__device__ __forceinline__ void quat_to_rot(const double* q, double R[9]) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1 - (txx + tyy);
}

__device__ __forceinline__ void load_pose(const double* p, double t[3], double q[4]) {
    t[0] = p[0]; t[1] = p[1]; t[2] = p[2];
    const double n = 1.0 / sqrt(p[3] * p[3] + p[4] * p[4] + p[5] * p[5] + p[6] * p[6]);  // SE3d(q, t) normalises
    q[0] = p[3] * n; q[1] = p[4] * n; q[2] = p[5] * n; q[3] = p[6] * n;
}

// SE3LeftParameterization::Plus: out = Sophus::SE3d::exp(delta) * (q, t)   (sophus/se3.hpp:763-784, so3.hpp:585-620)
__device__ __noinline__ void pose_plus(const double* pose, const double* d, double* out) {
    double t[3], q[4];
    load_pose(pose, t, q);
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
        double sh_, ch_;
        sincos(0.5 * theta, &sh_, &ch_);
        imag = sh_ / theta;
        real = ch_;
    }
    const double e[4] = {imag * ox, imag * oy, imag * oz, real};
    double Re[9];
    quat_to_rot(e, Re);
    double V[9];
    if (theta < SOPHUS_EPS) {
        for (int i = 0; i < 9; ++i) V[i] = Re[i];
    } else {
        const double a = (1.0 - cos(theta)) / th2;
        const double b = (theta - sin(theta)) / (th2 * theta);
        const double O[9] = {0, -oz, oy, oz, 0, -ox, -oy, ox, 0};
        double O2[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) O2[3 * i + j] = O[3 * i] * O[j] + O[3 * i + 1] * O[3 + j] + O[3 * i + 2] * O[6 + j];
        for (int i = 0; i < 9; ++i) V[i] = a * O[i] + b * O2[i];
        V[0] += 1.0; V[4] += 1.0; V[8] += 1.0;
    }
    const double et[3] = {V[0] * d[0] + V[1] * d[1] + V[2] * d[2], V[3] * d[0] + V[4] * d[1] + V[5] * d[2],
                          V[6] * d[0] + V[7] * d[1] + V[8] * d[2]};
    double r[4];   // quaternion product (so3.hpp:338-342), then normalisation
    r[3] = e[3] * q[3] - e[0] * q[0] - e[1] * q[1] - e[2] * q[2];
    r[0] = e[3] * q[0] + e[0] * q[3] + e[1] * q[2] - e[2] * q[1];
    r[1] = e[3] * q[1] + e[1] * q[3] + e[2] * q[0] - e[0] * q[2];
    r[2] = e[3] * q[2] + e[2] * q[3] + e[0] * q[1] - e[1] * q[0];
    const double n = 1.0 / sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
    out[0] = et[0] + Re[0] * t[0] + Re[1] * t[1] + Re[2] * t[2];
    out[1] = et[1] + Re[3] * t[0] + Re[4] * t[1] + Re[5] * t[2];
    out[2] = et[2] + Re[6] * t[0] + Re[7] * t[1] + Re[8] * t[2];
    out[3] = r[0] * n; out[4] = r[1] * n; out[5] = r[2] * n; out[6] = r[3] * n;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum(int v) { return __reduce_add_sync(FULL, v); }
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(FULL, v, o));
    return v;
}
__device__ __forceinline__ void atomic_max_pos(double* addr, double v) {
    // for non-negative doubles the bit pattern orders like an unsigned integer
    atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

// ------------------------------------------------------------------ barriers
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// Group barrier: monotonic arrival counter (zeroed by the host before the launch); barrier k completes when the
// counter reaches k * G.  Thread 0 arrives / spins, the rest of the CTA waits at the block barrier.  The gpu-scope
// fences publish this CTA's writes and invalidate its L1 (same construction as cooperative-groups grid.sync()).
// A spin that lasts ~seconds means a peer died: it raises `abort` (sticky) so that every later barrier falls
// through and the kernel drains instead of hanging the device.
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// OV2_BA_TRACE phase timer, run by one thread: mark(trace, k) charges the time since the previous mark to trace slot k
struct PhaseTimer {
    bool on;
    unsigned long long last;
    __device__ __forceinline__ explicit PhaseTimer(bool on_) : on(on_), last(on_ ? global_ns() : 0) {}
    __device__ __forceinline__ void mark(unsigned long long* trace, int k) {
        if (on) { const unsigned long long t = global_ns(); trace[k] += t - last; last = t; }
    }
};

constexpr unsigned long long BARRIER_TIMEOUT_NS = 30000000000ull;   // 30 s: a CTA that never arrives (includes waiting for CTA 0 inside a rank exchange)
constexpr unsigned long long XSYNC_TIMEOUT_NS = 20000000000ull;     // 20 s: a peer rank that never arrives

struct GroupBar {
    unsigned* count; unsigned* abort; unsigned G; unsigned epoch;
    __device__ __forceinline__ void sync() {
        __syncthreads();
        if (G > 1) {
            if (threadIdx.x == 0) {
                epoch += G;
                __threadfence();
                atomicAdd(count, 1u);
                unsigned spins = 0;
                unsigned long long t0 = 0;
                while (ld_acquire_gpu(count) < epoch) {
                    if ((++spins & 1023u) == 0) {
                        if (ld_acquire_gpu(abort)) break;
                        const unsigned long long t = global_ns();
                        if (t0 == 0) t0 = t;
                        else if (t - t0 > BARRIER_TIMEOUT_NS) { atomicExch(abort, 1u); break; }
                    }
                }
                __threadfence();
            }
            __syncthreads();
        }
    }
};

// ------------------------------------------------------------------ keyframe staging
// Rwc (9) + twc (3) of every keyframe of the window in the CTA's keyframe table: one normalisation + quaternion-to-rotation
// per keyframe and CTA instead of two per residual block.
__device__ __forceinline__ void cam_entry(const double* pose, double* e) {
    double t[3], q[4], R[9];
    load_pose(pose, t, q);
    quat_to_rot(q, R);
#pragma unroll
    for (int k = 0; k < 9; ++k) e[k] = R[k];
    e[9] = t[0]; e[10] = t[1]; e[11] = t[2];
}
__device__ __forceinline__ void stage_cams(const Prob& P, const double* __restrict__ pose, double* s_cam) {
    for (int c = threadIdx.x; c < P.ncam; c += blockDim.x) cam_entry(pose + 7 * c, s_cam + 12 * c);
}

// ------------------------------------------------------------------ residual blocks
// One residual block (src/ceres_parametrization.cpp:361-473 left camera; :579-712 right camera, other keyframe;
// :476-577 right camera in the anchor keyframe).  Returns the robustified cost 1/2 rho(s); writes chi2 / depth flag
// (the mutable members the reference's outlier scan reads afterwards) and, with JAC, the corrected Jacobian rows.
template <bool JAC>
__device__ __forceinline__ double eval_block(const Prob& P, int i, int lm, const double* __restrict__ s_cam, double lam, int use_huber) {
    const int ca = P.lm_anchor_cam[lm], co = P.obs_cam[i];
    const double* Rwa = s_cam + 12 * ca; const double* ta = Rwa + 9;
    const double* Rwc = s_cam + 12 * co; const double* to = Rwc + 9;
    const double zanch = 1.0 / lam;
    const double bx = (P.lm_anchor_px[2 * lm] - P.cx) / P.fx, by = (P.lm_anchor_px[2 * lm + 1] - P.cy) / P.fy;
    const double ap[3] = {zanch * bx, zanch * by, zanch};
    const double rp[3] = {Rwa[0] * ap[0] + Rwa[1] * ap[1] + Rwa[2] * ap[2], Rwa[3] * ap[0] + Rwa[4] * ap[1] + Rwa[5] * ap[2],
                          Rwa[6] * ap[0] + Rwa[7] * ap[1] + Rwa[8] * ap[2]};  // Rwanch * anchpt
    const double wp[3] = {rp[0] + ta[0], rp[1] + ta[1], rp[2] + ta[2]};
    const double dv[3] = {wp[0] - to[0], wp[1] - to[1], wp[2] - to[2]};
    const double lc[3] = {Rwc[0] * dv[0] + Rwc[3] * dv[1] + Rwc[6] * dv[2], Rwc[1] * dv[0] + Rwc[4] * dv[1] + Rwc[7] * dv[2],
                          Rwc[2] * dv[0] + Rwc[5] * dv[1] + Rwc[8] * dv[2]};   // Rcw = Rwc^T
    const int typ = P.obs_type ? (int)P.obs_type[i] : 0;
    double cp[3] = {lc[0], lc[1], lc[2]};
    double kfx = P.fx, kfy = P.fy, kcx = P.cx, kcy = P.cy;
    if (typ != 0) {
        const double* sv = typ == 2 ? ap : lc;
        for (int k = 0; k < 3; ++k) cp[k] = P.Rrl[3 * k] * sv[0] + P.Rrl[3 * k + 1] * sv[1] + P.Rrl[3 * k + 2] * sv[2] + P.trl[k];
        kfx = P.rfx; kfy = P.rfy; kcx = P.rcx; kcy = P.rcy;
    }
    const double linvz = 1.0 / cp[2];
    const double r0 = kfx * cp[0] * linvz + kcx - P.obs_px[2 * i];
    const double r1 = kfy * cp[1] * linvz + kcy - P.obs_px[2 * i + 1];
    const double s = r0 * r0 + r1 * r1;
    P.chi2[i] = s;
    P.dpos[i] = cp[2] > 0.0 ? 1 : 0;
    double w = 1.0, cost;
    if (use_huber && s > P.huber_b) {
        const double rs = sqrt(s);
        const double rho1 = fmax(DBL_MIN, P.huber_a / rs);
        cost = 0.5 * (2.0 * P.huber_a * rs - P.huber_b);
        w = sqrt(rho1);
    } else {
        cost = 0.5 * s;
    }
    if (JAC) {
        const double linvz2 = linvz * linvz;
        const double jc[6] = {linvz * kfx, 0.0, -cp[0] * linvz2 * kfx, 0.0, linvz * kfy, -cp[1] * linvz2 * kfy};
        // M = d(camera point)/d(world point): Rcw (left), Rrl Rcw (right, other frame), Rrl (right, anchor frame)
        double M[9];
        if (typ == 0) {
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) M[3 * a + b] = Rwc[3 * b + a];
        } else if (typ == 1) {
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    M[3 * a + b] = P.Rrl[3 * a] * Rwc[3 * b] + P.Rrl[3 * a + 1] * Rwc[3 * b + 1] + P.Rrl[3 * a + 2] * Rwc[3 * b + 2];
        } else {
            for (int k = 0; k < 9; ++k) M[k] = P.Rrl[k];
        }
        double JR[6];  // J_cam * M  (2x3)
        for (int a = 0; a < 2; ++a)
            for (int b = 0; b < 3; ++b)
                JR[3 * a + b] = jc[3 * a] * M[b] + jc[3 * a + 1] * M[3 + b] + jc[3 * a + 2] * M[6 + b];
        double JS[6];  // JR * hat(wpt)
        for (int a = 0; a < 2; ++a) {
            const double j0 = JR[3 * a], j1 = JR[3 * a + 1], j2 = JR[3 * a + 2];
            JS[3 * a] = j1 * wp[2] - j2 * wp[1];
            JS[3 * a + 1] = j2 * wp[0] - j0 * wp[2];
            JS[3 * a + 2] = j0 * wp[1] - j1 * wp[0];
        }
        double* Ja = P.Ja + 12 * (size_t)i;
        double* Jo = P.Jo + 12 * (size_t)i;
        const double wp_ = typ == 2 ? 0.0 : w;   // anchor-frame right-camera block: no pose block at all
        for (int a = 0; a < 2; ++a)
            for (int b = 0; b < 3; ++b) {
                Ja[6 * a + b] = wp_ * JR[3 * a + b];
                Ja[6 * a + 3 + b] = -wp_ * JS[3 * a + b];
                Jo[6 * a + b] = -wp_ * JR[3 * a + b];
                Jo[6 * a + 3 + b] = wp_ * JS[3 * a + b];
            }
        // J_lambda = -zanch * Rwanch * anchpt   (type 2: -zanch * anchpt, the point never leaves the anchor frame)
        const double* lp = typ == 2 ? ap : rp;
        const double jl[3] = {-zanch * lp[0], -zanch * lp[1], -zanch * lp[2]};
        P.Jl[2 * (size_t)i] = w * (JR[0] * jl[0] + JR[1] * jl[1] + JR[2] * jl[2]);
        P.Jl[2 * (size_t)i + 1] = w * (JR[3] * jl[0] + JR[4] * jl[1] + JR[5] * jl[2]);
        P.Jr[2 * (size_t)i] = w * r0;
        P.Jr[2 * (size_t)i + 1] = w * r1;
    }
    return cost;
}

// ------------------------------------------------------------------ Schur elimination (warp / landmark)

// Fire-and-forget fp64 add into GLOBAL memory.  atomicAdd(double*) on a generic pointer compiles to a run-time address-space
// test + ATOM.E.ADD.F64 (value returned) + a shared-memory CAS loop for the other branch; naming the state space gives one
// RED.E.ADD.F64 and nothing else.
__device__ __forceinline__ void red_add_f64(double* p, double v) {
    asm volatile("red.global.add.f64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "d"(v) : "memory");
}

// dst[j] += the CTA's sum of v[j], j < K: warp sums into the per-warp slots s_red, thread j adds the warps up in warp order
// and sends one RED per CTA (the CTAs of a group all hit the same addresses), none for a zero sum
template <int K, class T>
__device__ __forceinline__ void cta_red_add(const T (&v)[K], double (*s_red)[4], double* dst) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    T s[K];
#pragma unroll
    for (int j = 0; j < K; ++j) s[j] = warp_sum(v[j]);
    if (lane == 0)
#pragma unroll
        for (int j = 0; j < K; ++j) s_red[warp][j] = (double)s[j];
    __syncthreads();
    if (tid < K) {
        double a = 0.0;
        for (int w = 0; w < WARPS; ++w) a += s_red[w][tid];
        if (a != 0.0) red_add_f64(dst + tid, a);
    }
}

// LevenbergMarquardtStrategy (levenberg_marquardt_strategy.cc:66-160) with Jacobian scaling: column scale
// sc = 1 / (1 + sqrt(column norm)), fixed at the first iteration of a solve (`writer` stores it), and the damping term
// clamp(cn sc^2, 1e-6, 1e32) / (radius sc^2) added to the diagonal of the unscaled normal equations
__device__ __forceinline__ double lm_scale(double* stored, double cn, int first_iter, bool writer) {
    double sc = *stored;
    if (first_iter) {
        sc = 1.0 / (1.0 + sqrt(cn));
        if (writer) *stored = sc;
    }
    return sc;
}
__device__ __forceinline__ double lm_damping(double cn, double sc, double radius) {
    const double diag = fmin(fmax(cn * sc * sc, 1e-6), 1e32);
    return diag / (radius * sc * sc);
}

// schur_eliminator_impl.h:179-308 for a scalar e-block: E'E, E'r, F'F, F'r, E'F per touching keyframe, then
// S -= (E'F)' (E'E)^-1 (E'F), rhs -= (E'F)' (E'E)^-1 E'r.  The anchor keyframe's F'F / F'r / column norms are summed
// over the landmark's observations in registers and leave the warp once.
constexpr int SCH = 8;   // observations staged per chunk (C3: 4 per landmark, C5: 7.5)

// SM = false: contributions leave the warp as fp64 RED into the global accumulation block.  The phase is bound by the
// rate at which an SM retires fp64 REDs (it scales with 1/SMs, not with warps per SM), ~900 REDs per landmark.  SM = true
// (reduced systems that fit shared memory): `acc` is the warp's own copy of [rhs | F'r | column norms | S] in shared
// memory, updated with plain read-modify-writes (shared-memory fp64 atomics are CAS loops, slower than RED); the CTA sums
// its warps' copies and flushes the non-zeros once.
template <bool SM>
__device__ __forceinline__ void schur_landmark(const Prob& P, const int* __restrict__ s_slot, double* s_etf, int* s_eslot, double* sJ, int* smeta,
                                               int l, int lane, double radius, int first_iter, double* acc, int n, double& gmax_lm) {
#define ACC(ptr, v) do { if (SM) *(ptr) += (v); else red_add_f64((ptr), (v)); } while (0)
    const int p0 = P.lm_ptr[l], p1 = P.lm_ptr[l + 1];
    double* const cRhs = acc; double* const cG = acc + n; double* const cCn = acc + 2 * n; double* const cS = acc + 3 * n;
    double cnl = 0.0, ge = 0.0;
    int nact = 0;
    for (int p = p0 + lane; p < p1; p += 32) {
        const uint8_t act = P.active[p];                                   // loads issued together, selected after
        const double2 jl = *reinterpret_cast<const double2*>(P.Jl + 2 * (size_t)p);
        const double2 jr = *reinterpret_cast<const double2*>(P.Jr + 2 * (size_t)p);
        if (!act) continue;
        cnl += jl.x * jl.x + jl.y * jl.y;
        ge += jl.x * jr.x + jl.y * jr.y;
        nact++;
    }
    cnl = warp_sum(cnl);
    ge = warp_sum(ge);
    nact = __reduce_add_sync(FULL, nact);
    if (nact == 0) {   // unused parameter block: dropped from the program (program.cc:305-387)
        if (lane == 0) { P.ete[l] = 0.0; P.ge[l] = 0.0; }
        return;
    }
    const double sc = lm_scale(P.sc_lm + l, cnl, first_iter, lane == 0);
    const double ete = cnl + lm_damping(cnl, sc, radius);
    const double inv_ete = 1.0 / ete;
    if (lane == 0) {
        P.ete[l] = ete;
        P.ge[l] = ge;
    }
    gmax_lm = fmax(gmax_lm, fabs(ge));      // one atomicMax per warp and phase (per landmark they all hit ONE address: ~20 cycles each, serialised in L2)
    const int sa = s_slot[P.lm_anchor_cam[l]];
    int m = 0;   // number of E'F entries (uniform across the warp); entry 0 = anchor
    if (sa >= 0) {
        if (lane < 6) s_etf[lane] = 0.0;
        if (lane == 0) s_eslot[0] = sa;
        m = 1;
    }
    __syncwarp();
    // anchor accumulators: lane owns entries e = lane and lane + 32 of the 6x6 (a = e / 6, b = e % 6, a <= b kept)
    double aFF0 = 0.0, aFF1 = 0.0, aG = 0.0, aCn = 0.0, aE = 0.0;
    const int e0a = lane / 6, e0b = lane - 6 * e0a;
    const int e1 = lane + 32, e1a = e1 / 6, e1b = e1 - 6 * e1a;
    // The Jacobian rows of the landmark's observations are staged in this warp's shared-memory slice SCH at a time (coalesced
    // loads, all in flight together): the per-observation loop below then never waits on L2 (with one dependent global
    // load chain per observation and 8-16 warps per SM the phase was latency bound, 2.4x slower than the RED issue rate).
    double* sJa = sJ; double* sJo = sJ + 12 * SCH; double* sJl = sJ + 24 * SCH; double* sJr = sJ + 26 * SCH;
    for (int pb = p0; pb < p1; pb += SCH) {
        const int cnt = min(SCH, p1 - pb);
        __syncwarp();
        for (int e = lane; e < 12 * cnt; e += 32) { sJa[e] = P.Ja[12 * (size_t)pb + e]; sJo[e] = P.Jo[12 * (size_t)pb + e]; }
        if (lane < 2 * cnt) { sJl[lane] = P.Jl[2 * (size_t)pb + lane]; sJr[lane] = P.Jr[2 * (size_t)pb + lane]; }
        if (lane < cnt) {
            const int p = pb + lane;
            const uint8_t act = P.active[p], ty = P.obs_type ? P.obs_type[p] : 0;
            const int cam = P.obs_cam[p];
            smeta[lane] = !act ? -3 : (ty == 2 ? -2 : s_slot[cam]);   // -3: inactive, -2: e-block-only row (schur_eliminator_impl.h:196-217)
        }
        __syncwarp();
    for (int q = 0; q < cnt; ++q) {
        const int so = smeta[q];
        if (so < -1) continue;
        const double* Ja = sJa + 12 * q;
        const double* Jo = sJo + 12 * q;
        const double jl0 = sJl[2 * q], jl1 = sJl[2 * q + 1];
        const double r0 = sJr[2 * q], r1 = sJr[2 * q + 1];
        if (sa >= 0) {
            aFF0 += Ja[e0a] * Ja[e0b] + Ja[6 + e0a] * Ja[6 + e0b];
            if (e1 < 36) aFF1 += Ja[e1a] * Ja[e1b] + Ja[6 + e1a] * Ja[6 + e1b];
            if (lane < 6) {
                aG += Ja[lane] * r0 + Ja[6 + lane] * r1;
                aCn += Ja[lane] * Ja[lane] + Ja[6 + lane] * Ja[6 + lane];
                aE += jl0 * Ja[lane] + jl1 * Ja[6 + lane];
            }
        }
        if (so >= 0) {
            // E'F row of this keyframe: a stereo keyframe contributes two residual blocks (left and right camera) to the
            // same pose block, so look the slot up before appending a new entry
            int idx = -1;
            for (int qq = lane; qq < m; qq += 32)
                if (s_eslot[qq] == so) idx = qq;
            idx = __reduce_max_sync(FULL, idx);
            const bool fresh = idx < 0;
            if (fresh) idx = m;
            if (lane < 6) {
                const double e = jl0 * Jo[lane] + jl1 * Jo[6 + lane];
                s_etf[6 * idx + lane] = fresh ? e : s_etf[6 * idx + lane] + e;
            }
            if (lane == 0 && fresh) s_eslot[idx] = so;
            // The observation's six contributions per lane (observer diagonal block: 32 + 1 entries, F'r, column norms, cross
            // block Ja' Jo: 32 + 4 entries) go to DISTINCT addresses: addresses and values first, then all the loads, then all
            // the stores - the shared-memory mode pays one read-modify-write latency per observation instead of six.
            const int l6 = lane < 6 ? lane : 0, l4 = lane & 3;
            double* qp[6]; double qv[6]; bool qk[6];
            qk[0] = e0a <= e0b; qp[0] = cS + (size_t)(6 * so + e0a) * n + 6 * so + e0b; qv[0] = Jo[e0a] * Jo[e0b] + Jo[6 + e0a] * Jo[6 + e0b];
            qk[1] = lane == 3;  qp[1] = cS + (size_t)(6 * so + 5) * n + 6 * so + 5;     qv[1] = Jo[5] * Jo[5] + Jo[11] * Jo[11];
            qk[2] = lane < 6;   qp[2] = cG + 6 * so + l6;                               qv[2] = Jo[l6] * r0 + Jo[6 + l6] * r1;
            qk[3] = lane < 6;   qp[3] = cCn + 6 * so + l6;                              qv[3] = Jo[l6] * Jo[l6] + Jo[6 + l6] * Jo[6 + l6];
            // cross block Ja' Jo into the upper block (min slot, max slot); a: anchor column, b: observer column
            qk[4] = sa >= 0;             qv[4] = Ja[e0a] * Jo[e0b] + Ja[6 + e0a] * Jo[6 + e0b];
            qk[5] = sa >= 0 && lane < 4; qv[5] = Ja[5] * Jo[2 + l4] + Ja[11] * Jo[8 + l4];
            const int sa0 = sa >= 0 ? sa : 0;
            if (sa0 < so) { qp[4] = cS + (size_t)(6 * sa0 + e0a) * n + 6 * so + e0b; qp[5] = cS + (size_t)(6 * sa0 + 5) * n + 6 * so + 2 + l4; }
            else          { qp[4] = cS + (size_t)(6 * so + e0b) * n + 6 * sa0 + e0a; qp[5] = cS + (size_t)(6 * so + 2 + l4) * n + 6 * sa0 + 5; }
            if (SM) {
                double qo[6];
#pragma unroll
                for (int u = 0; u < 6; ++u) qo[u] = qk[u] ? *qp[u] : 0.0;
#pragma unroll
                for (int u = 0; u < 6; ++u) if (qk[u]) *qp[u] = qo[u] + qv[u];
            } else {
#pragma unroll
                for (int u = 0; u < 6; ++u) if (qk[u]) red_add_f64(qp[u], qv[u]);
            }
            if (fresh) m++;
        }
        __syncwarp();
    }
    }
    if (sa >= 0) {
        if (e0a <= e0b) ACC(cS + (size_t)(6 * sa + e0a) * n + 6 * sa + e0b, aFF0);
        if (e1 < 36 && e1a <= e1b) ACC(cS + (size_t)(6 * sa + e1a) * n + 6 * sa + e1b, aFF1);
        if (lane < 6) { ACC(cG + 6 * sa + lane, aG); ACC(cCn + 6 * sa + lane, aCn); }
    }
    if (sa >= 0 && lane < 6) s_etf[lane] += aE;     // the anchor's E'F row was summed in registers
    __syncwarp();
    // Schur complement: S[i,j] -= EtF_i' EtF_j / ete (upper blocks), rhs_i -= EtF_i ge / ete.  Pair-major: every unordered
    // pair of touching keyframes once, oriented by slot (the upper block), the 36 entries of a block on lanes 0..31 + a
    // second pass of 4 lanes - no per-entry divisions, no skipped iterations.
    {
        const int a0 = lane / 6, b0 = lane - 6 * a0;            // entry of pass 1
        const int a1 = 5, b1 = 2 + (lane & 3);                  // entries 32..35 of pass 2 (lanes 0..3)
        constexpr int U = 4;                                    // pairs per batch: 2 U independent read-modify-writes in flight
        const int npair = m * (m + 1) / 2;
        int i = 0, j = 0;
        for (int t0 = 0; t0 < npair; t0 += U) {
            double* q0[U]; double* q1[U]; double v0[U], v1[U]; bool k0[U], k1[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const bool live = t0 + u < npair;
                const int ii = live ? i : 0, jj = live ? j : 0;
                const int si = s_eslot[ii], sj = s_eslot[jj];
                const bool swap = si > sj;                      // block (lo, hi) with lo <= hi; entry (a, b) = etf_lo[a] etf_hi[b]
                const double* el = s_etf + 6 * (swap ? jj : ii);
                const double* eh = s_etf + 6 * (swap ? ii : jj);
                const int lo = swap ? sj : si, hi = swap ? si : sj;
                double* blkp = cS + (size_t)(6 * lo) * n + 6 * hi;
                q0[u] = blkp + (size_t)a0 * n + b0;
                q1[u] = blkp + (size_t)a1 * n + b1;
                k0[u] = live && (ii != jj || a0 <= b0);
                k1[u] = live && lane < 4 && (ii != jj || a1 <= b1);
                v0[u] = -(el[a0] * eh[b0] * inv_ete);
                v1[u] = -(el[a1] * eh[b1] * inv_ete);
                if (live && ++j == m) { ++i; j = i; }
            }
            if (SM) {
                double o0[U], o1[U];
#pragma unroll
                for (int u = 0; u < U; ++u) { o0[u] = k0[u] ? *q0[u] : 0.0; o1[u] = k1[u] ? *q1[u] : 0.0; }
#pragma unroll
                for (int u = 0; u < U; ++u) { if (k0[u]) *q0[u] = o0[u] + v0[u]; if (k1[u]) *q1[u] = o1[u] + v1[u]; }
            } else {
#pragma unroll
                for (int u = 0; u < U; ++u) { if (k0[u]) red_add_f64(q0[u], v0[u]); if (k1[u]) red_add_f64(q1[u], v1[u]); }
            }
        }
    }
    for (int e = lane; e < m * 6; e += 32) {
        const int i = e / 6, a = e - 6 * i;
        ACC(cRhs + 6 * s_eslot[i] + a, -s_etf[6 * i + a] * ge * inv_ete);
    }
    __syncwarp();
#undef ACC
}

// ------------------------------------------------------------------ Schur elimination, "owner" mode (reduced systems up to n = 96)
// The RED path above sends ~900 fp64 reductions per landmark to the global block, and an SM retires fp64 RED lanes at a
// few cycles each: in a batched C3 solve that phase dominates (OV2_BA_TRACE shows the split).  This mode forms the
// same sums where nothing has to be shared:
//   B1  camera part F'F, F'r, column norms: the observations are pre-sorted by (anchor keyframe, observing keyframe)
//       (host: pack_window), so a chunk of <= PCH observations touches ONE 12 x 12 Gram block [Ja | Jo]'[Ja | Jo]; a warp
//       owns a chunk, its lanes own the 78 + 12 entries (upper triangle + gradient), the chunk's Jacobian rows pass through the
//       warp's staging slice of shared memory, and the chunk's totals leave as <= 102 REDs (was ~89 per observation).
//   B2  landmark part: SG lanes per landmark form ete / g_e and the landmark's E'F row as a DENSE n-vector in a shared-memory
//       tile (one row per landmark, 32 / SG rows per warp); then S -= sum_rows w y y', rhs -= sum_rows w g_e y on the FP64
//       tensor cores, every warp owning 8 x 8 tiles of the upper triangle over ALL rounds (no atomics at all), flushed once.
constexpr int PCH = 32;           // observations per pair chunk

// FP64 tensor-core tile product (DMMA): D(8x8) = A(8x4) B(4x8) + C.  Fragment layout (PTX ISA, mma.m8n8k4 .f64):
// lane = 4 g + t; A: (row g, col t); B: (row t, col g); C/D: (row g, cols 2t, 2t+1).
__device__ __forceinline__ void dmma_884(double& d0, double& d1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
// pitch (doubles) of the owner-mode landmark tile: >= n rounded up to 8, congruent 4 mod 16
__host__ __device__ __forceinline__ int owner_tile_pitch(int n) {
    const int n8 = (n + 7) & ~7;
    return n8 + ((4 - n8) % 16 + 16) % 16;
}

template <int SG>
__device__ __forceinline__ void owner_fill_row(const Prob& P, const int* __restrict__ s_slot, int l, int sl, bool in, double radius, int first_iter,
                                               double* row, double& w_out, double& ge_out, double& gmax_lm) {
    const int p0 = in ? P.lm_ptr[l] : 0, p1 = in ? P.lm_ptr[l + 1] : 0;
    const int sa = in ? s_slot[P.lm_anchor_cam[l]] : -1;
    double cnl = 0.0, ge = 0.0, aE[6] = {0, 0, 0, 0, 0, 0};
    int nact = 0;
    for (int p = p0 + sl; p < p1; p += SG) {
        const uint8_t act = P.active[p];
        const double2 jl = *reinterpret_cast<const double2*>(P.Jl + 2 * (size_t)p);
        const double2 jr = *reinterpret_cast<const double2*>(P.Jr + 2 * (size_t)p);
        if (!act) continue;
        cnl += jl.x * jl.x + jl.y * jl.y;
        ge += jl.x * jr.x + jl.y * jr.y;
        nact++;
        if (P.obs_type && P.obs_type[p] == 2) continue;          // e-block-only row (schur_eliminator_impl.h:196-217)
        const double* Ja = P.Ja + 12 * (size_t)p;
        if (sa >= 0) {
#pragma unroll
            for (int k = 0; k < 6; ++k) aE[k] += jl.x * Ja[k] + jl.y * Ja[6 + k];
        }
        const int so = s_slot[P.obs_cam[p]];
        if (so >= 0) {
            const double* Jo = P.Jo + 12 * (size_t)p;
#pragma unroll
            for (int k = 0; k < 6; ++k) atomicAdd(row + 6 * so + k, jl.x * Jo[k] + jl.y * Jo[6 + k]);   // a stereo keyframe observes twice
        }
    }
#pragma unroll
    for (int o = SG / 2; o > 0; o >>= 1) {
        cnl += __shfl_xor_sync(FULL, cnl, o);
        ge += __shfl_xor_sync(FULL, ge, o);
        nact += __shfl_xor_sync(FULL, nact, o);
#pragma unroll
        for (int k = 0; k < 6; ++k) aE[k] += __shfl_xor_sync(FULL, aE[k], o);
    }
    w_out = 0.0;
    ge_out = 0.0;
    if (!in) return;
    if (nact == 0) {   // unused parameter block: dropped from the program (program.cc:305-387)
        if (sl == 0) { P.ete[l] = 0.0; P.ge[l] = 0.0; }
        return;
    }
    const double sc = lm_scale(P.sc_lm + l, cnl, first_iter, sl == 0);
    const double ete = cnl + lm_damping(cnl, sc, radius);
    if (sl == 0) {
        P.ete[l] = ete;
        P.ge[l] = ge;
        if (sa >= 0) {
#pragma unroll
            for (int k = 0; k < 6; ++k) atomicAdd(row + 6 * sa + k, aE[k]);
        }
    }
    gmax_lm = fmax(gmax_lm, fabs(ge));
    w_out = 1.0 / ete;
    ge_out = ge;
}

template <int NT, int SG>
__device__ __noinline__ void schur_owner_phase(const Prob& P, const int* __restrict__ s_slot, double* s_tile, int n, double radius, int first_iter,
                                               int bid, int G, double* scal) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gwarps = G * WARPS, gwarp = bid * WARPS + warp;
    double* const cRhs = P.acc; double* const cG = P.acc + n; double* const cCn = P.acc + 2 * n; double* const cS = P.acc + 3 * n;
    // ---------------- B1: camera part, one pair chunk per warp
    PhaseTimer tm(P.trace != nullptr && bid == 0 && tid == 0);
    {
        double* st = s_tile + (size_t)warp * (PCH * 26);
        int ia0[3], ja0[3], ja1[3], ei[3], ej[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int e = lane + 32 * k;
            ei[k] = -1; ej[k] = -1; ia0[k] = 0; ja0[k] = 0; ja1[k] = 0;
            if (e < 78) {
                int i = 0, rem = e;
                while (rem >= 12 - i) { rem -= 12 - i; ++i; }
                const int j = i + rem;
                ei[k] = i; ej[k] = j;
                ia0[k] = i < 6 ? i : i + 6;
                ja0[k] = j < 6 ? j : j + 6;
                ja1[k] = ja0[k] + 6;
            } else if (e < 90) {
                const int i = e - 78;
                ei[k] = i; ej[k] = 12;                              // gradient entry: [Ja | Jo]' r
                ia0[k] = i < 6 ? i : i + 6;
                ja0[k] = 24; ja1[k] = 25;
            }
        }
        for (int c = gwarp; c < P.npchunk; c += gwarps) {
            const int2 ch = P.pair_chunk[c];
            const int cnt = ch.y - ch.x;                             // <= PCH = 32: lane q looks after observation q
            int pq = 0, onq = 0;
            if (lane < cnt) {
                pq = P.pair_perm[ch.x + lane];
                onq = (P.active[pq] && !(P.obs_type && P.obs_type[pq] == 2)) ? 1 : 0;
            }
            const int pf = __shfl_sync(FULL, pq, 0);
            const int sa = s_slot[P.lm_anchor_cam[P.obs_lm[pf]]], so = s_slot[P.obs_cam[pf]];
            if (sa < 0 && so < 0) continue;                         // both keyframes constant / unused (warp-uniform)
            // the whole chunk's rows [Ja | Jo | r] go to this warp's staging slice with every load in flight at once (staging
            // four observations at a time left the phase waiting on one L2 round trip per stage: 4.1 ms of a batched C3 solve)
            __syncwarp();
            // (two unrolled halves of 13 loads per lane: every load of a half is issued before the first store needs its value -
            //  a rolled load -> store loop waited one L2 round trip per element, 14.6 us per chunk)
            const int tot = cnt * 26;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                double vals[13];
#pragma unroll
                for (int j = 0; j < 13; ++j) {
                    const int e = (half * 13 + j) * 32 + lane;
                    const bool ok = e < tot;
                    const int q = ok ? e / 26 : 0, k = e - 26 * q;
                    const int p = __shfl_sync(FULL, pq, q);
                    const int on = __shfl_sync(FULL, onq, q);
                    const double* src = k < 12 ? P.Ja + 12 * (size_t)p + k : (k < 24 ? P.Jo + 12 * (size_t)p + (k - 12) : P.Jr + 2 * (size_t)p + (k - 24));
                    vals[j] = (ok && on) ? *src : 0.0;
                }
#pragma unroll
                for (int j = 0; j < 13; ++j) {
                    const int e = (half * 13 + j) * 32 + lane;
                    if (e < tot) st[e] = vals[j];
                }
            }
            __syncwarp();
            double a[3] = {0.0, 0.0, 0.0};
            for (int q = 0; q < cnt; ++q) {
                const double* v = st + 26 * q;
#pragma unroll
                for (int k = 0; k < 3; ++k) a[k] += v[ia0[k]] * v[ja0[k]] + v[ia0[k] + 6] * v[ja1[k]];
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int i = ei[k], j = ej[k];
                double v = a[k];
                if (i < 0 || v == 0.0) continue;
                if (j == 12) {                                      // F'r
                    if (i < 6) { if (sa >= 0) red_add_f64(cG + 6 * sa + i, v); }
                    else if (so >= 0) red_add_f64(cG + 6 * so + (i - 6), v);
                } else if (j < 6) {                                 // anchor diagonal block (i <= j < 6)
                    if (sa >= 0) {
                        red_add_f64(cS + (size_t)(6 * sa + i) * n + 6 * sa + j, v);
                        if (i == j) red_add_f64(cCn + 6 * sa + i, v);
                    }
                } else if (i >= 6) {                                // observer diagonal block
                    if (so >= 0) {
                        red_add_f64(cS + (size_t)(6 * so + (i - 6)) * n + 6 * so + (j - 6), v);
                        if (i == j) red_add_f64(cCn + 6 * so + (i - 6), v);
                    }
                } else if (sa >= 0 && so >= 0) {                    // cross block Ja' Jo into the upper block (min slot, max slot)
                    const int ca = i, cb = j - 6;
                    if (sa < so) red_add_f64(cS + (size_t)(6 * sa + ca) * n + 6 * so + cb, v);
                    else if (sa > so) red_add_f64(cS + (size_t)(6 * so + cb) * n + 6 * sa + ca, v);
                    else {                                          // same pose block twice: Ja'Jo + Jo'Ja lands in its diagonal block
                        if (ca == cb) { v *= 2.0; red_add_f64(cCn + 6 * sa + ca, v); }
                        const int lo = ca < cb ? ca : cb, hi = ca < cb ? cb : ca;
                        red_add_f64(cS + (size_t)(6 * sa + lo) * n + 6 * sa + hi, v);
                    }
                }
            }
        }
    }
    __syncthreads();
    tm.mark(P.trace, 15);                                           // trace slot 15 = B1 share of B:schur in this mode
    // ---------------- B2: landmark part
    // S -= sum_rows w y y' is the one contraction of this phase: FP64 tensor cores (DMMA m8n8k4), a warp owns up to NT 8 x 8
    // tiles of the upper triangle and keeps their accumulators in registers over ALL rounds; per 4-row step and tile two
    // shared-memory loads (tile pitch = 4 mod 16 doubles: conflict-free half-warps) and one DMMA.
    constexpr int R = WARPS * (32 / SG);                            // tile rows (landmarks per round and CTA)
    const int TP = owner_tile_pitch(n);
    double* tw = s_tile + (size_t)R * TP;
    double* tg = tw + R;
    const int nb8 = (n + 7) >> 3, ntile = nb8 * (nb8 + 1) / 2;
    int bi[NT], bj[NT];
    double acc[NT][2];
#pragma unroll
    for (int k = 0; k < NT; ++k) {
        const int t = warp + WARPS * k;
        bi[k] = -1; bj[k] = 0;
        if (t < ntile) {
            int i = 0, rem = t;
            while (rem >= nb8 - i) { rem -= nb8 - i; ++i; }
            bi[k] = i; bj[k] = i + rem;
        }
        acc[k][0] = 0.0; acc[k][1] = 0.0;
    }
    double racc = 0.0, gmax_lm = 0.0;
    const int sub = lane / SG, sl = lane - sub * SG;
    const int myrow = warp * (32 / SG) + sub;
    const int fg = lane >> 2, ft = lane & 3;                        // DMMA fragment coordinates
    for (int l0 = bid * R; l0 < P.npts; l0 += G * R) {
        for (int e = tid; e < R * TP + 2 * R; e += THREADS) s_tile[e] = 0.0;
        __syncthreads();
        {
            const int l = l0 + myrow;
            double w, g;
            owner_fill_row<SG>(P, s_slot, l, sl, l < P.npts, radius, first_iter, s_tile + (size_t)myrow * TP, w, g, gmax_lm);
            if (sl == 0) { tw[myrow] = w; tg[myrow] = g; }
        }
        __syncthreads();
        const int rows = min(R, P.npts - l0);
        for (int k0 = 0; k0 < rows; k0 += 4) {                      // rows beyond `rows` are zero rows with w = 0
            const double* yk = s_tile + (size_t)(k0 + ft) * TP;
            const double wv = tw[k0 + ft];
#pragma unroll
            for (int k = 0; k < NT; ++k) {
                if (bi[k] < 0) continue;                            // warp-uniform
                dmma_884(acc[k][0], acc[k][1], yk[8 * bi[k] + fg] * wv, yk[8 * bj[k] + fg]);
            }
        }
        if (tid < n) {
            double ra = 0.0;
            for (int r = 0; r < rows; ++r) ra += s_tile[(size_t)r * TP + tid] * (tw[r] * tg[r]);
            racc -= ra;
        }
        __syncthreads();
    }
    // flush: every upper-triangle entry of this CTA's partial system has exactly one owner
#pragma unroll
    for (int k = 0; k < NT; ++k) {
        if (bi[k] < 0) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int r = 8 * bi[k] + fg, c = 8 * bj[k] + 2 * ft + e;
            const double v = acc[k][e];
            if (r <= c && c < n && v != 0.0) red_add_f64(cS + (size_t)r * n + c, -v);
        }
    }
    if (tid < n && racc != 0.0) red_add_f64(cRhs + tid, racc);
    gmax_lm = warp_max(gmax_lm);
    if (lane == 0 && gmax_lm > 0.0) atomic_max_pos(scal + SC_GMAX_LM, gmax_lm);
}

// ------------------------------------------------------------------ reduced camera system, n <= 96: CTA-wide Gauss-Jordan in shared memory
// Augmented system [S + D | b] in shared memory (row pitch n + 2); pivot step j updates every row r != j for the columns
// c > j: A[r][c] -= (A[r][j] / A[j][j]) A[j][c].  Row j and column j are not written in step j, so ONE block barrier per
// pivot suffices and no substitution passes follow (a Cholesky + two triangular solves is 3n dependent steps).  Pivots
// equal those of the LDL' / Cholesky factorisation (no pivoting: S is SPD after LM damping), so "pivot <= 0" is the
// failure test Ceres' LLT applies.  Four threads per row; a thread stages the pivot-row and own-row entries of its
// columns in registers first (all shared-memory loads in flight together), then updates and stores.
template <int QMAX>
__device__ __forceinline__ void gj_pivots(double* sA, int n, int PIT, int* s_fail) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int sub = tid & 3, r0 = tid >> 2, rows_per_pass = nt >> 2;
    for (int j = 0; j < n; ++j) {
        const double p = sA[j * PIT + j];
        if (!(p > 0.0) || !isfinite(p)) { if (tid == 0) *s_fail = 1; break; }   // uniform: every thread reads the same pivot
        // 1 / p sits on the critical path of every pivot (tens of cycles per DEPENDENT fp64 operation - the 48-pivot loop
        // is latency bound on this chain): MUFU double-precision seed (2^-23) + two Newton steps, no float round trip
        double ip;
        asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(ip) : "d"(p));
        ip = fma(ip, fma(-p, ip, 1.0), ip);
        ip = fma(ip, fma(-p, ip, 1.0), ip);
        const double* rowj = sA + j * PIT;
        const int c0 = j + 1 + sub;
        const int nq = (n - j + 3 - sub) >> 2;              // columns c = c0 + 4 q <= n
        double pj[QMAX];
#pragma unroll
        for (int q = 0; q < QMAX; ++q) pj[q] = q < nq ? rowj[c0 + 4 * q] : 0.0;
        for (int r = r0; r < n; r += rows_per_pass) {
            if (r == j) continue;
            double* rowr = sA + r * PIT;
            const double f = rowr[j] * ip;
            double a[QMAX];
#pragma unroll
            for (int q = 0; q < QMAX; ++q) a[q] = q < nq ? rowr[c0 + 4 * q] : 0.0;
#pragma unroll
            for (int q = 0; q < QMAX; ++q) a[q] -= f * pj[q];
#pragma unroll
            for (int q = 0; q < QMAX; ++q)
                if (q < nq) rowr[c0 + 4 * q] = a[q];
        }
        __syncthreads();
    }
}

__device__ void reduced_solve_small(const Prob& P, double* T, int n, double radius, int first_iter, double* sA, double* scal) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int PIT = n + 2;
    PhaseTimer tm(P.trace != nullptr && tid == 0);              // (CTA 0 only runs this) trace slots 12: load + damping, 13: pivots, 14: solution
    double* cRhs = T; double* cG = T + n; double* cCn = T + 2 * n; double* cS = T + 3 * n;
    __shared__ int s_fail;
    if (tid == 0) s_fail = 0;
    for (int e = tid; e < n * n; e += nt) {
        const int r = e / n, c = e - r * n;
        sA[r * PIT + c] = r <= c ? cS[(size_t)r * n + c] : cS[(size_t)c * n + r];
    }
    __syncthreads();
    for (int i = tid; i < n; i += nt) {
        const double cn = cCn[i];
        const double sc = lm_scale(P.sc_cam + i, cn, first_iter, true);
        sA[i * PIT + i] += lm_damping(cn, sc, radius);
        sA[i * PIT + n] = cG[i] + cRhs[i];
    }
    __syncthreads();
    tm.mark(P.trace, 12);
    if (n <= 48) gj_pivots<13>(sA, n, PIT, &s_fail);         // (n + 1 + 3) / 4 columns per thread
    else if (n <= 64) gj_pivots<17>(sA, n, PIT, &s_fail);
    else gj_pivots<25>(sA, n, PIT, &s_fail);
    __syncthreads();
    tm.mark(P.trace, 13);
    if (s_fail) {
        if (tid == 0) scal[SC_CHOL_FAIL] = 1.0;
        return;
    }
    for (int i = tid; i < n; i += nt) P.z[i] = sA[i * PIT + n] / sA[i * PIT + i];
    tm.mark(P.trace, 14);
}

// ------------------------------------------------------------------ reduced camera system, n > 96: blocked Cholesky across the group
// Right-looking blocked Cholesky in blocks of CH_NB.  Only the sequential part of a block step stays on CTA 0 (diagonal
// block, row panel, forward substitution); the trailing update A22 -= U12' U12 - the one real contraction, (n - c1)^2 x 32
// flops - is spread over every warp of the group (FP64 tensor cores, operands read from the row panel in L2).  Two group
// barriers per block step; 9 steps for the 288 x 288 system of a 48-keyframe window.
__device__ void reduced_solve_blocked_group(const Prob& P, double* T, int n, double radius, int first_iter, double* sP, double* scal,
                                            GroupBar& bar, int bid, int G) {
    const int tid = threadIdx.x, nt = blockDim.x;
    double* cRhs = T; double* cG = T + n; double* cCn = T + 2 * n; double* A = T + 3 * n;
    __shared__ double s_w[MAX_N];
    __shared__ double sU[CH_NB][CH_NB + 1];
    __shared__ double s_idiag_all[MAX_N + CH_NB];
    __shared__ double s_t[CH_NB];
    __shared__ int s_bad;
    double* w = s_w;
    const int PW = ((n + 15) & ~15) + 8;                 // row pitch of the panel (doubles)
    double* Pan = P.panel;                               // [CH_NB][PW] in global memory: what the other CTAs read
    const int warp = tid >> 5, lane = tid & 31, nwarp = nt >> 5;
    const int gwarps = G * nwarp, gwarp = bid * nwarp + warp;
    PhaseTimer tm(P.trace != nullptr && bid == 0 && tid == 0);
    if (bid == 0) {
        if (tid == 0) s_bad = 0;
        for (int i = tid; i < n; i += nt) {
            const double cn = cCn[i];
            const double sc = lm_scale(P.sc_cam + i, cn, first_iter, true);
            A[(size_t)i * n + i] += lm_damping(cn, sc, radius);
            w[i] = cG[i] + cRhs[i];
        }
        __syncthreads();
    }
    for (int kb = 0; kb < n; kb += CH_NB) {
        const int nb = min(CH_NB, n - kb), c1 = kb + nb, m = n - c1;
        const int m16 = (m + 15) & ~15;
        if (bid == 0) {
            double* s_idiag = s_idiag_all + kb;
            for (int e = tid; e < CH_NB * CH_NB; e += nt) {
                const int i = e >> 5, j = e & 31;
                sU[i][j] = (i < nb && j < nb && i <= j) ? A[(size_t)(kb + i) * n + kb + j] : (i == j ? 1.0 : 0.0);
            }
            __syncthreads();
            if (warp == 0) {
                // One warp, lane = column, the column's 32 rows in REGISTERS (fully unrolled): per pivot the dependent
                // chain is shuffle -> MUFU rsqrt seed + two Newton steps -> scale -> one shared-memory row broadcast ->
                // 31 independent FMAs.  (The shared-memory read-modify-write form this replaces serialised ~16 row
                // updates per pivot on the ~50-cycle fp64 latency: 1.5 k cycles per pivot, 25 us per block step.)
                bool bad = false;
                double a[CH_NB];
#pragma unroll
                for (int r = 0; r < CH_NB; ++r) a[r] = sU[r][lane];
#pragma unroll
                for (int j = 0; j < CH_NB; ++j) {
                    const double d = __shfl_sync(FULL, a[j], j);
                    bad = bad || !(d > 1e-30) || !(d < 1e30);
                    double is;
                    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(is) : "d"(d));
                    is = fma(0.5 * is, fma(-d * is, is, 1.0), is);
                    is = fma(0.5 * is, fma(-d * is, is, 1.0), is);
                    const double ujc = lane >= j ? a[j] * is : 0.0;
                    sU[j][lane] = ujc;                     // row j of U: final value, and the broadcast source below
                    if (lane == j) s_idiag[j] = is;
                    __syncwarp();
                    // (measured alternatives, both slower: broadcasting U[j][r] by shuffle - no warp barrier in the chain, but
                    // 62 SHFL per pivot: +40 %; for the Gauss-Jordan above, forming the next pivot's reciprocal one step ahead,
                    // redundantly in every thread or in a dedicated warp: +10 % - the pivot chain is not what bounds a step)
#pragma unroll
                    for (int r = j + 1; r < CH_NB; ++r) a[r] = fma(-sU[j][r], ujc, a[r]);   // entries below the diagonal (r > lane) are never read
                }
                if (bad && lane == 0) { s_bad = 1; scal[SC_CHOL_FAIL] = 1.0; }
            }
            __syncthreads();
            if (!s_bad) {
                for (int e = tid; e < CH_NB * CH_NB; e += nt) {
                    const int i = e >> 5, j = e & 31;
                    if (i < nb && j < nb && i <= j) A[(size_t)(kb + i) * n + kb + j] = sU[i][j];
                }
                for (int cc = tid; cc <= m16; cc += nt) {
                    if (cc >= m && cc < m16) {                                   // zero padding of the operand panel
#pragma unroll
                        for (int i = 0; i < CH_NB; ++i) { sP[i * PW + cc] = 0.0; Pan[i * PW + cc] = 0.0; }
                        continue;
                    }
                    const bool is_rhs = cc == m16;
                    if (!is_rhs && cc >= m) continue;
                    double a[CH_NB];
#pragma unroll
                    for (int i = 0; i < CH_NB; ++i)
                        a[i] = i < nb ? (is_rhs ? w[kb + i] : A[(size_t)(kb + i) * n + c1 + cc]) : 0.0;
#pragma unroll
                    for (int k = 0; k < CH_NB; ++k) {
                        const double x = a[k] * s_idiag[k];
                        a[k] = x;
#pragma unroll
                        for (int i = k + 1; i < CH_NB; ++i) a[i] -= sU[k][i] * x;
                    }
                    if (is_rhs) {
#pragma unroll
                        for (int i = 0; i < CH_NB; ++i) if (i < nb) { w[kb + i] = a[i]; s_t[i] = a[i]; }
                    } else {
#pragma unroll
                        for (int i = 0; i < CH_NB; ++i) {
                            sP[i * PW + cc] = a[i];
                            Pan[i * PW + cc] = a[i];
                            if (i < nb) A[(size_t)(kb + i) * n + c1 + cc] = a[i];
                        }
                    }
                }
            }
        }
        tm.mark(P.trace, 12);
        bar.sync();
        tm.mark(P.trace, 13);
        if (scal[SC_CHOL_FAIL] != 0.0) return;                           // uniform across the group (written before the barrier)
        if (bid == 0) {
            for (int r = tid; r < m; r += nt) {
                double acc = 0.0;
#pragma unroll 8
                for (int k = 0; k < CH_NB; ++k) acc += sP[k * PW + r] * s_t[k];
                w[c1 + r] -= acc;
            }
        }
        {
            const int mt = m16 >> 4, g = lane >> 2, t = lane & 3;
            for (int idx = gwarp; idx < mt * mt; idx += gwarps) {
                const int tr = idx / mt, tc = idx - tr * mt;
                if (tr > tc) continue;
                const int r0 = tr * 16, q0 = tc * 16;
                double acc[2][2][2] = {{{0.0, 0.0}, {0.0, 0.0}}, {{0.0, 0.0}, {0.0, 0.0}}};
#pragma unroll
                for (int k0 = 0; k0 < CH_NB; k0 += 4) {
                    const double* pk = Pan + (size_t)(k0 + t) * PW;
                    const double a0 = pk[r0 + g], a1 = pk[r0 + 8 + g];
                    const double b0 = pk[q0 + g], b1 = pk[q0 + 8 + g];
                    dmma_884(acc[0][0][0], acc[0][0][1], a0, b0);
                    dmma_884(acc[0][1][0], acc[0][1][1], a0, b1);
                    dmma_884(acc[1][0][0], acc[1][0][1], a1, b0);
                    dmma_884(acc[1][1][0], acc[1][1][1], a1, b1);
                }
#pragma unroll
                for (int hi = 0; hi < 2; ++hi)
#pragma unroll
                    for (int hj = 0; hj < 2; ++hj)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int r = r0 + 8 * hi + g, c = q0 + 8 * hj + 2 * t + e;
                            if (r <= c && c < m) A[(size_t)(c1 + r) * n + c1 + c] -= acc[hi][hj][e];
                        }
            }
        }
        tm.mark(P.trace, 14);
        bar.sync();
        tm.mark(P.trace, 13);
    }
    if (bid != 0) return;
    // ---- backward substitution U z = y, last block first (CTA 0)
    for (int kb = ((n - 1) / CH_NB) * CH_NB; kb >= 0; kb -= CH_NB) {
        const int nb = min(CH_NB, n - kb), c1 = kb + nb;
        for (int e = tid; e < CH_NB * CH_NB; e += nt) {
            const int i = e >> 5, j = e & 31;
            sU[i][j] = (i < nb && j < nb && i <= j) ? A[(size_t)(kb + i) * n + kb + j] : (i == j ? 1.0 : 0.0);
        }
        for (int i = warp; i < nb; i += nwarp) {
            double acc = 0.0;
            for (int c = c1 + lane; c < n; c += 32) acc += A[(size_t)(kb + i) * n + c] * w[c];
            acc = warp_sum(acc);
            if (lane == 0) s_t[i] = w[kb + i] - acc;
        }
        __syncthreads();
        if (warp == 0) {
            double ti = lane < nb ? s_t[lane] : 0.0;
            const double idg = lane < nb ? s_idiag_all[kb + lane] : 1.0;
#pragma unroll
            for (int j = CH_NB - 1; j >= 0; --j) {
                const double zj = __shfl_sync(FULL, ti * idg, j);
                if (lane < j) ti -= sU[lane][j] * zj;
                if (lane == j && j < nb) w[kb + j] = zj;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < n; i += nt) P.z[i] = w[i];
    tm.mark(P.trace, 15);
}

// ------------------------------------------------------------------ back-substitution + candidate cost (SG lanes / landmark)
// schur_eliminator_impl.h:311-377: y_e = (E'E)^-1 (E'r - sum_k (E'F_k) z_k); model cost change
// -(J delta)'(r + J delta / 2) (trust_region_minimizer.cc:424-427); candidate inverse depth; then the residual blocks of
// the landmark at the candidate point (cost only).
// SG lanes per landmark, 32 / SG landmarks per warp in flight (SG = 4 / 8 for windows with few observations per landmark).
// A landmark has ~4 (C3) to ~8 (C5) observations, so one warp per landmark leaves most lanes idle and - worse - strings the
// landmarks' dependent load chains (CSR pointers -> Jacobian rows -> reduction -> second pass) one after the other:
// measured 3.9 ms of a 11.9 ms batched C3 solve.  The per-landmark sums are formed inside the sub-group.
template <int SG>
__device__ __forceinline__ void backsub_landmarks_sg(const Prob& P, const int* __restrict__ s_slot, const double* __restrict__ s_cam,
                                                     int l0, int lane, const double* __restrict__ invd, double* __restrict__ cand_invd,
                                                     int use_huber, double& mcc_out, double& st2_out, double& cx2_out, double& cost_out) {
    const int sub = lane / SG, sl = lane - sub * SG;
    const int l = l0 + sub;
    const bool in = l < P.npts;
    const double ete = in ? P.ete[l] : 0.0;
    const bool live = in && ete != 0.0;     // ete == 0: landmark not in the program, candidate stays equal
    const int p0 = live ? P.lm_ptr[l] : 0, p1 = live ? P.lm_ptr[l + 1] : 0;
    const int sa = live ? s_slot[P.lm_anchor_cam[l]] : -1;
    double za[6] = {0, 0, 0, 0, 0, 0};
    if (sa >= 0)
        for (int k = 0; k < 6; ++k) za[k] = P.z[6 * sa + k];
    double acc = 0.0;
    for (int p = p0 + sl; p < p1; p += SG) {
        if (!P.active[p]) continue;
        const int so = (P.obs_type && P.obs_type[p] == 2) ? -1 : s_slot[P.obs_cam[p]];
        const double* Ja = P.Ja + 12 * (size_t)p;
        const double* Jo = P.Jo + 12 * (size_t)p;
        double f0 = 0.0, f1 = 0.0;
        if (sa >= 0)
            for (int k = 0; k < 6; ++k) { f0 += Ja[k] * za[k]; f1 += Ja[6 + k] * za[k]; }
        if (so >= 0)
            for (int k = 0; k < 6; ++k) { const double zk = P.z[6 * so + k]; f0 += Jo[k] * zk; f1 += Jo[6 + k] * zk; }
        acc += P.Jl[2 * (size_t)p] * f0 + P.Jl[2 * (size_t)p + 1] * f1;
    }
#pragma unroll
    for (int o = SG / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
    const double y = live ? (P.ge[l] - acc) / ete : 0.0;
    const double dl = -y;
    const double cl = live ? invd[l] + dl : 0.0;
    double mcc = 0.0, cost = 0.0;
    for (int p = p0 + sl; p < p1; p += SG) {
        if (!P.active[p]) continue;
        const int so = (P.obs_type && P.obs_type[p] == 2) ? -1 : s_slot[P.obs_cam[p]];
        const double* Ja = P.Ja + 12 * (size_t)p;
        const double* Jo = P.Jo + 12 * (size_t)p;
        double f0 = P.Jl[2 * (size_t)p] * dl, f1 = P.Jl[2 * (size_t)p + 1] * dl;
        if (sa >= 0)
            for (int k = 0; k < 6; ++k) { f0 -= Ja[k] * za[k]; f1 -= Ja[6 + k] * za[k]; }
        if (so >= 0)
            for (int k = 0; k < 6; ++k) { const double zk = P.z[6 * so + k]; f0 -= Jo[k] * zk; f1 -= Jo[6 + k] * zk; }
        mcc -= f0 * (P.Jr[2 * (size_t)p] + 0.5 * f0) + f1 * (P.Jr[2 * (size_t)p + 1] + 0.5 * f1);
        cost += eval_block<false>(P, p, l, s_cam, cl, use_huber);
    }
    if (live && sl == 0) {
        cand_invd[l] = cl;
        st2_out += dl * dl;
        cx2_out += cl * cl;
    }
    mcc_out += mcc;
    cost_out += cost;
}

// ------------------------------------------------------------------ multi-GPU exchange (peer memory over NVLink)
// Every rank exports one buffer (see ba_lm.cuh); xsync() is a barrier between the ranks' kernels: CTA 0 / thread 0
// writes its epoch into slot `rank` of every peer's flag array (release, system scope) and waits until every peer
// has written the same epoch into ours.  Must be bracketed by group barriers.
__device__ __forceinline__ void xsync(const Peers& X, unsigned long long& xepoch, unsigned* abort) {
    xepoch++;
    __threadfence_system();
    for (int r = 0; r < X.world; ++r)
        if (r != X.rank) st_release_sys(reinterpret_cast<unsigned long long*>(X.base[r]) + X.rank, xepoch);
    for (int r = 0; r < X.world; ++r) {
        if (r == X.rank) continue;
        const unsigned long long* f = reinterpret_cast<const unsigned long long*>(X.base[X.rank]) + r;
        unsigned spins = 0;
        unsigned long long t0 = 0;
        while (ld_acquire_sys(f) < xepoch) {
            if ((++spins & 255u) == 0) {
                if (ld_acquire_gpu(abort)) break;
                const unsigned long long t = global_ns();
                if (t0 == 0) t0 = t;
                else if (t - t0 > XSYNC_TIMEOUT_NS) { atomicExch(abort, 1u); break; }
            }
        }
    }
    __threadfence_system();
}

__device__ __forceinline__ double ld_peer(const double* p) {
    double v;
    asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

// rank r's part of the exchange buffer from byte offset `off` (an XB_* offset) on, as mapped in this process
template <class T>
__device__ __forceinline__ T* xslice(const Peers& X, int r, size_t off) {
    return reinterpret_cast<T*>(static_cast<unsigned char*>(X.base[r]) + off);
}

// One exchange between the ranks: `publish` writes this rank's slice, then group barrier, xsync on CTA 0 / thread 0, group
// barrier.  Afterwards every rank's slice is readable.  Every rank's kernel runs the same sequence of exchanges.
template <class F>
__device__ __forceinline__ void rank_exchange(const Peers& X, GroupBar& bar, int bid, unsigned long long& xepoch, F publish) {
    publish();
    bar.sync();
    if (bid == 0 && threadIdx.x == 0) xsync(X, xepoch, bar.abort);
    bar.sync();
}

// ------------------------------------------------------------------ the persistent solve kernel
struct SolveOut { int iterations; double initial_cost, final_cost; int termination; };

__global__ void __launch_bounds__(THREADS, 2) ba_lm_kernel(const Prob* __restrict__ probs, int nprob, int G, Peers X) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ lmctl::State S;
    __shared__ int s_action, s_ncv, s_any, s_refine, s_trivial;
    __shared__ double s_red[WARPS][4];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int group = blockIdx.x / G, bid = blockIdx.x - group * G, ngroups = gridDim.x / G;
    if (group >= ngroups) return;
    unsigned long long xepoch = X.epoch0;
    __shared__ Prob sProb;
    for (int pi = group; pi < nprob; pi += ngroups) {
        __syncthreads();
        for (int i = tid; i < (int)(sizeof(Prob) / sizeof(int)); i += THREADS)
            reinterpret_cast<int*>(&sProb)[i] = reinterpret_cast<const int*>(probs + pi)[i];
        __syncthreads();
        const Prob& P = sProb;
        GroupBar bar{P.bar, P.bar + 1, (unsigned)G, 0u};
        // trace slots 0-11 (the kernel's phases) add up in tr_acc and are stored at the end: a read-modify-write of the global
        // trace per mark costs the kernel registers
        unsigned long long tr_acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        PhaseTimer tm(P.trace != nullptr && bid == 0 && tid == 0);
        // keyframe table [ncam][12] + [ncam] slots: in shared memory, or (windows too large for it) this CTA's copy in
        // global memory; either way only this CTA reads and writes it
        double* s_cam = P.cam_tab ? P.cam_tab + (size_t)bid * P.cam_tab_stride : reinterpret_cast<double*>(smem_raw);
        int* s_slot = reinterpret_cast<int*>(s_cam + 12 * (size_t)P.ncam);
        double* s_work = reinterpret_cast<double*>(smem_raw + P.smem_work_off);    // Schur scratch / solve area (union)
        const int etf_stride = 6 * (P.ncv_max + 1);
        double* s_etf = s_work + (size_t)warp * etf_stride;
        int* s_eslot = reinterpret_cast<int*>(s_work + (size_t)WARPS * etf_stride) + warp * (P.ncv_max + 1);
        double* sJ = s_work + (size_t)WARPS * etf_stride + (((size_t)WARPS * (P.ncv_max + 1) + 1) >> 1) + (size_t)warp * (28 * SCH);
        int* smeta = reinterpret_cast<int*>(s_work + (size_t)WARPS * etf_stride + (((size_t)WARPS * (P.ncv_max + 1) + 1) >> 1) + (size_t)WARPS * (28 * SCH)) + warp * SCH;
        const int gthreads = G * THREADS, gtid = bid * THREADS + tid;
        const int gwarps = G * WARPS, gwarp = bid * WARPS + warp;
        const size_t blk = P.blk;                                                  // doubles per accumulation copy (n_max based)
        int xi = 0;                                                                // index of the buffer holding x
        int use_huber = P.use_robust;
        int n_out1 = 0, n_out2 = 0;
        SolveOut so[2];
        so[0] = SolveOut{0, 0.0, 0.0, 0};
        so[1] = SolveOut{0, 0.0, 0.0, 0};
        int ran_refine = 0;
        for (int stage = 0; stage < 2; ++stage) {
            const int max_iters = stage == 0 ? P.max_it1 : P.max_it2;
            uint8_t* cam_used = P.cam_used + (size_t)stage * P.ncam;
            double* x_pose = P.pose[xi]; double* c_pose = P.pose[xi ^ 1];
            double* x_invd = P.invd[xi]; double* c_invd = P.invd[xi ^ 1];
            // ---- set-up: Program::RemoveFixedBlocks (keyframes that are constant or touch no active residual drop out),
            //      candidate := x for the blocks that are not in this solve's program, accumulators zeroed
            // (flags are collected per CTA in shared memory first: thousands of stores from every SM to the same few bytes
            //  serialise in L2 - measured 7 us per CTA of the group)
            for (int c = tid; c < P.ncam; c += THREADS) s_slot[c] = 0;
            __syncthreads();
            for (int i = gtid; i < P.nobs; i += gthreads)
                if (P.active[i] && !(P.obs_type && P.obs_type[i] == 2)) {
                    s_slot[P.obs_cam[i]] = 1;
                    s_slot[P.lm_anchor_cam[P.obs_lm[i]]] = 1;
                }
            __syncthreads();
            for (int c = tid; c < P.ncam; c += THREADS)
                if (s_slot[c]) cam_used[c] = 1;
            for (int i = gtid; i < 7 * P.ncam; i += gthreads) c_pose[i] = x_pose[i];
            for (int i = gtid; i < P.npts; i += gthreads) c_invd[i] = x_invd[i];
            for (size_t i = gtid; i < blk; i += gthreads) P.acc[i] = 0.0;
            for (int i = gtid; i < 2 * SC_COUNT; i += gthreads) P.scal[i] = 0.0;
            tm.mark(tr_acc, stage == 0 ? 0 : 10);
            bar.sync();
            tm.mark(tr_acc, stage == 0 ? 11 : 10);
            if (X.world > 1) {
                // a keyframe is in the program if ANY rank has an active residual touching it
                const size_t xb = XB_CAMUSED + (size_t)stage * MAX_CAMS;
                rank_exchange(X, bar, bid, xepoch, [&] {
                    uint8_t* mine = xslice<uint8_t>(X, X.rank, xb);
                    for (int i = gtid; i < P.ncam; i += gthreads) mine[i] = cam_used[i];
                });
                for (int c = tid; c < P.ncam; c += THREADS) {
                    int u = 0;
                    for (int r = 0; r < X.world; ++r) u |= xslice<volatile const uint8_t>(X, r, xb)[c];
                    s_slot[c] = (u ? 1 : 0) | (P.pose_const[c] ? 2 : 0);          // temporarily: used / constant flags
                }
            } else {
                for (int c = tid; c < P.ncam; c += THREADS) s_slot[c] = (cam_used[c] ? 1 : 0) | (P.pose_const[c] ? 2 : 0);
            }
            __syncthreads();
            if (tid == 0) {
                int ncv = 0, any = 0;
                for (int c = 0; c < P.ncam; ++c) {
                    const int u = s_slot[c];
                    any |= u & 1;
                    s_slot[c] = u == 1 ? ncv++ : -1;
                }
                s_ncv = ncv; s_any = any;
                lmctl::init(S);
            }
            __syncthreads();
            const int ncv = s_ncv, n = 6 * ncv;
            if (!s_any) { if (stage == 0) break; else continue; }   // no residual blocks (on any rank)
            if (bid == 0)
                for (int c = tid; c < P.ncam; c += THREADS) P.cam_slot[c] = s_slot[c];
            double* T = X.world > 1 ? P.total : P.acc;                       // the system the solve reads
            tm.mark(tr_acc, 0);
            // ---- LM iterations
            for (;;) {
                if (tid == 0) s_action = lmctl::begin_iteration(S, max_iters) ? 1 : 0;
                __syncthreads();
                if (!s_action) break;
                const int par = S.iteration & 1, first_iter = S.first_iter, x_is_new = S.x_is_new;
                const double radius = S.radius;
                double* scal = P.scal + par * SC_COUNT;
                // ---- A: residual blocks + Jacobians at x
                if (x_is_new) {
                    stage_cams(P, x_pose, s_cam);
                    __syncthreads();
                    double cost[1] = {0.0};
                    for (int i = gtid; i < P.nobs; i += gthreads)
                        if (P.active[i]) cost[0] += eval_block<true>(P, i, P.obs_lm[i], s_cam, x_invd[P.obs_lm[i]], use_huber);
                    cta_red_add(cost, s_red, scal + SC_COST);
                }
                bar.sync();
                tm.mark(tr_acc, 1);
                // ---- B: Schur elimination into the accumulation block
                if (P.schur_smem == 3) {
                    // owner mode (n <= 96): pair-sorted Gram blocks + dense landmark rows, no per-observation reductions
#define OV2_OWNER(NT_) do { if (P.sg == 4) schur_owner_phase<NT_, 4>(P, s_slot, s_work, n, radius, first_iter, bid, G, scal); \
                            else if (P.sg == 8) schur_owner_phase<NT_, 8>(P, s_slot, s_work, n, radius, first_iter, bid, G, scal); \
                            else schur_owner_phase<NT_, 32>(P, s_slot, s_work, n, radius, first_iter, bid, G, scal); } while (0)
                    if (n <= 48) OV2_OWNER(3);            // 21 upper 8 x 8 tiles over 8 warps
                    else if (n <= 72) OV2_OWNER(6);       // 45
                    else OV2_OWNER(10);                   // 78 (n = 96)
#undef OV2_OWNER
                } else if (P.schur_smem == 2) {
                    // per-WARP private copies of [rhs | F'r | column norms | S] in shared memory: plain read-modify-writes, no
                    // lock, no RED; the CTA sums its copies and sends the non-zeros to the global block once per phase
                    const int live_s = 3 * n + n * n;
                    double* mine = s_work + P.smem_sacc_off + (size_t)warp * live_s;
                    for (int e = lane; e < live_s; e += 32) mine[e] = 0.0;
                    __syncwarp();
                    double gmax_lm = 0.0;
                    for (int l = gwarp; l < P.npts; l += gwarps) schur_landmark<true>(P, s_slot, s_etf, s_eslot, sJ, smeta, l, lane, radius, first_iter, mine, n, gmax_lm);
                    if (lane == 0 && gmax_lm > 0.0) atomic_max_pos(scal + SC_GMAX_LM, gmax_lm);
                    __syncthreads();
                    const double* all = s_work + P.smem_sacc_off;
                    for (int e = tid; e < live_s; e += THREADS) {
                        double v = 0.0;
#pragma unroll
                        for (int w_ = 0; w_ < WARPS; ++w_) v += all[(size_t)w_ * live_s + e];
                        if (v != 0.0) red_add_f64(P.acc + e, v);
                    }
                } else {
                    double gmax_lm = 0.0;
                    for (int l = gwarp; l < P.npts; l += gwarps) schur_landmark<false>(P, s_slot, s_etf, s_eslot, sJ, smeta, l, lane, radius, first_iter, P.acc, n, gmax_lm);
                    if (lane == 0 && gmax_lm > 0.0) atomic_max_pos(scal + SC_GMAX_LM, gmax_lm);
                }
                bar.sync();
                tm.mark(tr_acc, 2);
                // ---- B2: multi-GPU: sum the ranks' partial systems out of peer memory
                const int live = 3 * n + n * n;
                if (X.world > 1) {
                    const size_t slot = (size_t)par * (SC_COUNT + blk);   // [scalars | partial system] of this parity
                    rank_exchange(X, bar, bid, xepoch, [&] {
                        double* mine = xslice<double>(X, X.rank, XB_PARTIAL) + slot;
                        for (int e = gtid; e < live; e += gthreads) mine[SC_COUNT + e] = P.acc[e];
                        if (gtid < SC_COUNT) mine[gtid] = scal[gtid];
                    });
                    for (int e = gtid; e < live; e += gthreads) {
                        double a = 0.0;
                        for (int r = 0; r < X.world; ++r) a += ld_peer(xslice<const double>(X, r, XB_PARTIAL) + slot + SC_COUNT + e);
                        T[e] = a;
                    }
                    if (gtid == 0) {
                        double c = 0.0, g = 0.0;
                        for (int r = 0; r < X.world; ++r) {
                            const double* pr = xslice<const double>(X, r, XB_PARTIAL) + slot;
                            c += ld_peer(pr + SC_COST);
                            g = fmax(g, ld_peer(pr + SC_GMAX_LM));
                        }
                        scal[SC_COST] = c;        // the whole window's cost / gradient bound, identical on every rank
                        scal[SC_GMAX_LM] = g;
                    }
                    bar.sync();
                }
                tm.mark(tr_acc, 3);
                // ---- C: reduced camera system (CTA 0); gradient projection |x - Plus(x, -g)|_inf (last CTA); the other
                //      CTAs clear the accumulation block for the next iteration once the solve has read it
                const bool group_solve = P.solve_blocked && n > 0;
                if (bid == 0 && !group_solve && n > 0) reduced_solve_small(P, T, n, radius, first_iter, s_work, scal);
                if (bid == G - 1 && x_is_new && n > 0) {
                    if (bid == 0) __syncthreads();
                    double gm = 0.0;
                    for (int c = tid; c < P.ncam; c += THREADS) {
                        const int s = s_slot[c];
                        if (s < 0) continue;
                        double d[6], out[7];
                        for (int k = 0; k < 6; ++k) d[k] = -T[n + 6 * s + k];
                        pose_plus(x_pose + 7 * c, d, out);
                        for (int k = 0; k < 7; ++k) gm = fmax(gm, fabs(x_pose[7 * c + k] - out[k]));
                    }
                    gm = warp_max(gm);
                    if (lane == 0) atomic_max_pos(scal + SC_GMAX_CAM, gm);
                }
                if (group_solve) reduced_solve_blocked_group(P, T, n, radius, first_iter, s_work, scal, bar, bid, G);
                tm.mark(tr_acc, 4);
                bar.sync();
                tm.mark(tr_acc, 5);
                // ---- D: candidate keyframe poses (every CTA, into shared memory), back-substitution, candidate cost
                {
                    double st2 = 0.0, cx2 = 0.0;
                    for (int c = tid; c < P.ncam; c += THREADS) {
                        const int s = s_slot[c];
                        double out[7];
                        if (s >= 0) {
                            double d[6];
                            for (int k = 0; k < 6; ++k) d[k] = -P.z[6 * s + k];
                            pose_plus(x_pose + 7 * c, d, out);
                            for (int k = 0; k < 7; ++k) {
                                const double df = x_pose[7 * c + k] - out[k];
                                st2 += df * df; cx2 += out[k] * out[k];
                            }
                            if (bid == 0)
                                for (int k = 0; k < 7; ++k) c_pose[7 * c + k] = out[k];
                        } else {
                            for (int k = 0; k < 7; ++k) out[k] = x_pose[7 * c + k];
                        }
                        cam_entry(out, s_cam + 12 * c);
                    }
                    __syncthreads();
                    double mcc = 0.0, cost = 0.0, lst2 = 0.0, lcx2 = 0.0;
#define OV2_BACKSUB(SG_) for (int l0 = gwarp * (32 / SG_); l0 < P.npts; l0 += gwarps * (32 / SG_)) \
                             backsub_landmarks_sg<SG_>(P, s_slot, s_cam, l0, lane, x_invd, c_invd, use_huber, mcc, lst2, lcx2, cost)
                    if (P.sg == 4) OV2_BACKSUB(4);
                    else if (P.sg == 8) OV2_BACKSUB(8);
                    else OV2_BACKSUB(32);
#undef OV2_BACKSUB
                    // the keyframe part of the norms counts once per window (rank 0, CTA 0)
                    if (bid == 0 && X.rank == 0) { lst2 += st2; lcx2 += cx2; }
                    const double sums[4] = {cost, mcc, lst2, lcx2};   // SC_CAND_COST, SC_MCC, SC_STEP2, SC_CANDX2
                    cta_red_add(sums, s_red, scal + SC_CAND_COST);
                    // clear for the next iteration: accumulation block and the other parity's scalars
                    for (size_t i = gtid; i < blk; i += gthreads) P.acc[i] = 0.0;
                    double* oscal = P.scal + (par ^ 1) * SC_COUNT;
                    if (gtid < SC_COUNT) oscal[gtid] = 0.0;
                }
                bar.sync();
                tm.mark(tr_acc, 6);
                if (X.world > 1) {
                    // second, tiny exchange: candidate cost, model cost change, step / candidate norms (rank order sum)
                    rank_exchange(X, bar, bid, xepoch, [&] {
                        if (gtid < 4) xslice<double>(X, X.rank, XB_SC4)[par * 8 + gtid] = scal[SC_CAND_COST + gtid];
                    });
                }
                // ---- E: trust-region controller, replayed by every CTA
                if (tid == 0) {
                    double v[4];
                    if (X.world > 1) {
                        for (int k = 0; k < 4; ++k) {
                            double a = 0.0;
                            for (int r = 0; r < X.world; ++r) a += ld_peer(xslice<const double>(X, r, XB_SC4) + par * 8 + k);
                            v[k] = a;
                        }
                    } else {
                        for (int k = 0; k < 4; ++k) v[k] = scal[SC_CAND_COST + k];
                    }
                    const double gmax = fmax(scal[SC_GMAX_LM], scal[SC_GMAX_CAM]);
                    s_action = (int)lmctl::end_iteration(S, scal[SC_COST], v[0], v[1], v[2], v[3], gmax, scal[SC_CHOL_FAIL] != 0.0, P.ftol);
                }
                __syncthreads();
                const int action = s_action;
                tm.mark(tr_acc, 7);
                if (action == lmctl::ACT_CONTINUE_ACCEPTED) {
                    xi ^= 1;
                    x_pose = P.pose[xi]; c_pose = P.pose[xi ^ 1];
                    x_invd = P.invd[xi]; c_invd = P.invd[xi ^ 1];
                }
                if (action == lmctl::ACT_STOP) break;
            }
            so[stage].iterations = S.iteration;
            so[stage].initial_cost = S.initial_cost;
            so[stage].final_cost = lmctl::final_cost(S);
            so[stage].termination = S.termination;
            if (stage == 1) ran_refine = 1;
            // a stop while a candidate was pending leaves buffers unequal for out-of-program blocks only at the
            // next set-up (which copies x over the candidate), so nothing to repair here
            bar.sync();
            // ---- outlier scan on the values the LAST evaluation left behind (optimizer.cpp:500-530, :637-735)
            {
                double* cnt = P.counts + 4 * stage;
                const int bit = stage == 0 ? 1 : 2;
                const int deact = stage == 0 && P.apply_l2;
                int nt[3] = {0, 0, 0};                           // outliers, left-camera and right-camera inliers
                for (int i = gtid; i < P.nobs; i += gthreads) {
                    if (!P.active[i]) continue;
                    const bool bad = (P.chi2[i] > (double)P.th_f) || !P.dpos[i];
                    if (bad) {
                        P.flags[i] |= (uint8_t)bit;
                        if (deact) P.active[i] = 0;   // problem.RemoveResidualBlock
                        nt[0]++;
                    } else {
                        const int typ = P.obs_type ? (int)P.obs_type[i] : 0;
                        nt[1] += typ == 0;
                        nt[2] += typ == 1;
                    }
                }
                cta_red_add(nt, s_red, cnt);
                // the stop request lives in mapped HOST memory: ONE thread of the group reads it (every thread of every CTA
                // polling it over PCIe cost 7 us per CTA of the group) and publishes it next to the counters
                if (stage == 0 && bid == 0 && tid == 0)
                    cnt[3] = (P.stop_flag && *reinterpret_cast<volatile const int*>(P.stop_flag) != 0) ? 1.0 : 0.0;
                bar.sync();
                if (stage == 0) {
                    double nbad = cnt[0], nleft = cnt[1], nright = cnt[2];
                    n_out1 = (int)nbad;
                    if (X.world > 1) {
                        // every rank must take the same branch: counts summed over the ranks
                        rank_exchange(X, bar, bid, xepoch, [&] {
                            if (gtid < 3) xslice<double>(X, X.rank, XB_SC4)[16 + gtid] = cnt[gtid];
                        });
                        nbad = nleft = nright = 0.0;
                        for (int r = 0; r < X.world; ++r) {
                            const double* pr = xslice<const double>(X, r, XB_SC4) + 16;
                            nbad += ld_peer(pr); nleft += ld_peer(pr + 1); nright += ld_peer(pr + 2);
                        }
                    }
                    // solve #2 only if residual blocks were removed and no stop was requested meanwhile (optimizer.cpp:603-604)
                    int refine = P.apply_l2 && P.use_robust && nbad > 0.0;
                    if (refine && cnt[3] != 0.0) refine = 0;        // (sharded callers pass no stop flag: ranks could disagree)
                    // mono windows keep the Huber loss in the refinement; the wrapper is reset to the trivial loss only when
                    // left-camera and other-frame right-camera residual lists are both non-empty (optimizer.cpp:606-608)
                    int trivial = P.refine_loss;
                    if (trivial < 0) trivial = (nleft > 0.0 && nright > 0.0) ? 1 : 0;
                    if (tid == 0) { s_refine = refine; s_trivial = trivial; }
                    __syncthreads();
                    if (!s_refine) break;
                    use_huber = s_trivial ? 0 : 1;
                } else {
                    n_out2 = (int)cnt[0];
                }
            }
        }
        // ---- write-back: x into buffer 0, result record
        tm.mark(tr_acc, 8);
        bar.sync();
        if (xi == 1) {
            for (int i = gtid; i < 7 * P.ncam; i += gthreads) P.pose[0][i] = P.pose[1][i];
            for (int i = gtid; i < P.npts; i += gthreads) P.invd[0][i] = P.invd[1][i];
        }
        if (bid == 0 && tid == 0) {
            Result* R = P.result;
            R->iters_robust = so[0].iterations;
            R->iters_refine = ran_refine ? so[1].iterations : 0;
            const SolveOut& last = ran_refine ? so[1] : so[0];
            R->initial_cost = last.initial_cost;
            R->final_cost = last.final_cost;
            R->termination = last.termination;
            R->n_outliers_first = n_out1;
            R->n_outliers_second = n_out2;
            R->aborted = (int)ld_acquire_gpu(P.bar + 1);
        }
        tm.mark(tr_acc, 9);
        if (tm.on)
            for (int k = 0; k < 12; ++k) P.trace[k] = tr_acc[k];
    }
}

}  // namespace balm

// ====================================================================== host side
using namespace balm;

namespace {

// The memory of one batch in regions, every window's arrays side by side in each.  Device blocks:
//   upload block [state | input]: one H2D; state first, so one D2H brings the poses and inverse depths of every window back
//   work block   [work | zero | output | active]: one memset each for zero + output and for active, one D2H of output
// The pinned host block mirrors [state | input | output].  A window's arrays are taken while it is planned, as offsets
// inside their region; place() fixes the regions once every window is planned, and d() / h() give the addresses.
enum Region { RG_STATE, RG_INPUT, RG_WORK, RG_ZERO, RG_OUT, RG_ACT, RG_COUNT };

struct Span { Region rg; size_t off; };

struct Layout {
    size_t used[RG_COUNT] = {};
    char* dev[RG_COUNT] = {};
    char* host[RG_COUNT] = {};   // state, input and output regions only

    Span take(Region rg, size_t bytes, size_t align = 256) {
        size_t& u = used[rg];
        u = (u + align - 1) & ~(align - 1);
        const Span sp{rg, u};
        u += bytes;
        return sp;
    }
    size_t bytes(Region rg) const { return (used[rg] + 255) & ~(size_t)255; }
    size_t upload_bytes() const { return bytes(RG_STATE) + bytes(RG_INPUT); }
    size_t work_bytes() const { return bytes(RG_WORK) + bytes(RG_ZERO) + bytes(RG_OUT) + bytes(RG_ACT); }
    void place(char* upload, char* work, char* pinned) {
        dev[RG_STATE] = upload;
        dev[RG_INPUT] = upload + bytes(RG_STATE);
        dev[RG_WORK] = work;
        for (int r = RG_ZERO; r < RG_COUNT; ++r) dev[r] = dev[r - 1] + bytes((Region)(r - 1));
        host[RG_STATE] = pinned;
        host[RG_INPUT] = pinned + bytes(RG_STATE);
        host[RG_OUT] = pinned + upload_bytes();
    }
    char* d(Span sp) const { return dev[sp.rg] + sp.off; }
    char* h(Span sp) const { return host[sp.rg] + sp.off; }
};

struct HostPlan {
    Span pose, invd;                                                               // state
    Span prob, apx, opx, lac, oc, ol, lp, pc, ty, pp, pch;                        // input
    Span pose1, invd1, camslot, Jr, Ja, Jo, Jl, chi2, dpos, ete, ge, acc, total, scal, z, panel, camtab;   // work
    Span camused, counts, bar, trace, sclm, sccam;                                // zero
    Span result, flags;                                                            // output
    Span active;                                                                   // active
    int pch_cap, sg;   // owner mode: chunk table capacity (pp: pair-sorted permutation, pch: chunk table); lanes per landmark
    int ncv_max, n_max, solve_blocked, schur_smem;
    bool cam_tab_global;                     // keyframe table in the work block (one copy per CTA), not in shared memory
    size_t blk, tab_bytes, smem_work_off, smem_bytes, smem_sacc_off;
};

// Where a window's arrays live.  A window whose `pose` array is host memory is taken to be host memory throughout (the
// reference's flow, optimizer.cpp:43-430): cudaPointerGetAttributes costs ~1.5 us on a plain host pointer, and 15 queries
// per window were 6 ms of a 296-window batch.  Only windows whose poses live on the device are inspected array by array.
struct Residence {
    bool window = false;            // `pose` is device memory
    bool invd = false, flags = false;
    bool on_device(const void* p) const { return window && p && ov2_is_device_ptr(p); }
};

// a state array between the caller's memory and the pinned block
cudaError_t copy_state(void* dst, const void* src, size_t bytes, bool device, cudaMemcpyKind kind) {
    if (bytes == 0) return cudaSuccess;
    if (device) return cudaMemcpy(dst, src, bytes, kind);
    memcpy(dst, src, bytes);
    return cudaSuccess;
}

}  // namespace

// Plans one window: its arrays in the batch's regions, its Schur mode, reduced solver and shared-memory layout.
static ov2_status plan_window(ov2_ctx* ctx, const ov2_ba_problem* pb, int world, Layout& L, HostPlan& H, bool single_window) {
    const int ncam = pb->ncam, npts = pb->npts, nobs = pb->nobs;
    int ncv = 0;
    for (int c = 0; c < ncam; ++c) ncv += pb->pose_const[c] ? 0 : 1;
    if (world == 1 && ncv > 0) {
        // Optimised keyframes are the non-constant ones some pose-dependent residual touches as observer or anchor
        // (Program::RemoveFixedBlocks drops the others; the kernel's rule in each stage).  Every residual starts active and
        // the active set only shrinks, so this count bounds both stages.  A rank of a multi-GPU window sees only its own
        // shard and keeps the declared count.  The scan stops once every declared keyframe has been seen.
        std::vector<uint8_t> seen((size_t)ncam, 0);
        int nused = 0;
        for (int i = 0; i < nobs && nused < ncv; ++i) {
            if (pb->obs_type && pb->obs_type[i] == 2) continue;
            const int l = pb->obs_lm[i];
            if (l < 0 || l >= npts) continue;                          // refused when the window is packed
            for (const int c : {pb->obs_cam[i], pb->lm_anchor_cam[l]})
                if (c >= 0 && c < ncam && !pb->pose_const[c] && !seen[c]) { seen[c] = 1; ++nused; }
        }
        ncv = nused;
    }
    if (ncv > MAX_VAR_CAMS) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_localba_solve: more than 64 optimised keyframes");
    if (world > 1 && ncam > MAX_CAMS) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_localba_solve_p2p: more than 256 keyframes in a multi-GPU window");
    H.ncv_max = ncv; H.n_max = 6 * ncv;
    H.blk = 3 * (size_t)H.n_max + (size_t)H.n_max * H.n_max;
    if (H.blk == 0) H.blk = 1;
    H.solve_blocked = H.n_max > 96 ? 1 : 0;
    // states (pose, inverse depth) of all windows sit together at the head of the block: they are what comes back
    H.pose = L.take(RG_STATE, sizeof(double) * 7 * ncam, 16);
    H.invd = L.take(RG_STATE, sizeof(double) * (size_t)(npts > 0 ? npts : 1), 16);
    H.prob = L.take(RG_INPUT, sizeof(Prob));
    H.apx = L.take(RG_INPUT, sizeof(double) * 2 * (size_t)(npts > 0 ? npts : 1));
    H.opx = L.take(RG_INPUT, sizeof(double) * 2 * (size_t)(nobs > 0 ? nobs : 1));
    H.lac = L.take(RG_INPUT, sizeof(int32_t) * (size_t)(npts > 0 ? npts : 1));
    H.oc = L.take(RG_INPUT, sizeof(int32_t) * (size_t)(nobs > 0 ? nobs : 1));
    H.ol = L.take(RG_INPUT, sizeof(int32_t) * (size_t)(nobs > 0 ? nobs : 1));
    H.lp = L.take(RG_INPUT, sizeof(int32_t) * (size_t)(npts + 1));
    H.pc = L.take(RG_INPUT, (size_t)ncam);
    H.ty = L.take(RG_INPUT, pb->obs_type ? (size_t)(nobs > 0 ? nobs : 1) : 0);
    {
        // owner-mode Schur (n <= 96): observations sorted by (anchor keyframe, observing keyframe) + chunk table
        const size_t ngmax = (size_t)ncam * ncam < (size_t)(nobs > 0 ? nobs : 1) ? (size_t)ncam * ncam : (size_t)(nobs > 0 ? nobs : 1);
        H.pch_cap = (int)((size_t)(nobs > 0 ? nobs : 1) / PCH + ngmax + 1);
        H.pp = L.take(RG_INPUT, sizeof(int32_t) * (size_t)(nobs > 0 ? nobs : 1));
        H.pch = L.take(RG_INPUT, sizeof(int2) * (size_t)H.pch_cap);
        const double avg = npts > 0 ? (double)nobs / (double)npts : 0.0;
        H.sg = avg <= 5.0 ? 4 : (avg <= 12.0 ? 8 : 32);
    }
    const size_t no = nobs > 0 ? nobs : 1, np = npts > 0 ? npts : 1;
    H.result = L.take(RG_OUT, sizeof(Result), 64);
    H.flags = L.take(RG_OUT, no, 64);
    H.active = L.take(RG_ACT, no, 64);
    H.camused = L.take(RG_ZERO, 2 * (size_t)ncam);
    H.counts = L.take(RG_ZERO, sizeof(double) * 8);
    H.bar = L.take(RG_ZERO, sizeof(unsigned) * 4);
    H.trace = L.take(RG_ZERO, sizeof(unsigned long long) * 16);
    H.sclm = L.take(RG_ZERO, sizeof(double) * np);
    H.sccam = L.take(RG_ZERO, sizeof(double) * MAX_N);
    H.pose1 = L.take(RG_WORK, sizeof(double) * 7 * ncam);
    H.invd1 = L.take(RG_WORK, sizeof(double) * np);
    H.camslot = L.take(RG_WORK, sizeof(int32_t) * ncam);
    H.Jr = L.take(RG_WORK, sizeof(double) * 2 * no);
    H.Ja = L.take(RG_WORK, sizeof(double) * 12 * no);
    H.Jo = L.take(RG_WORK, sizeof(double) * 12 * no);
    H.Jl = L.take(RG_WORK, sizeof(double) * 2 * no);
    H.chi2 = L.take(RG_WORK, sizeof(double) * no);
    H.dpos = L.take(RG_WORK, no);
    H.ete = L.take(RG_WORK, sizeof(double) * np);
    H.ge = L.take(RG_WORK, sizeof(double) * np);
    H.acc = L.take(RG_WORK, sizeof(double) * H.blk);
    H.total = L.take(RG_WORK, sizeof(double) * H.blk);
    H.scal = L.take(RG_WORK, sizeof(double) * 2 * SC_COUNT);
    H.z = L.take(RG_WORK, sizeof(double) * MAX_N);
    H.panel = L.take(RG_WORK, sizeof(double) * CH_NB * (size_t)(MAX_N + 24));
    // dynamic shared memory: [keyframe table: 12 doubles + 1 slot each][union: Schur scratch | solve area]
    size_t s = sizeof(double) * 12 * (size_t)ncam + sizeof(int) * (size_t)ncam;
    s = (s + 15) & ~(size_t)15;
    H.tab_bytes = s;
    H.smem_work_off = s;
    size_t schur = (size_t)WARPS * 6 * (size_t)(ncv + 1) * sizeof(double) + ((((size_t)WARPS * (ncv + 1) + 1) >> 1) << 3) +
                   (size_t)WARPS * 28 * SCH * sizeof(double) + (size_t)WARPS * SCH * sizeof(int) + 16;
    schur = (schur + 15) & ~(size_t)15;
    const size_t solve = H.solve_blocked ? (size_t)CH_NB * (size_t)((((size_t)H.n_max + 15) & ~(size_t)15) + 8) * sizeof(double)
                                         : (size_t)H.n_max * (size_t)(H.n_max + 2) * sizeof(double);
    // shared-memory accumulation of the reduced system (behind the Schur scratch) when the whole block fits next to it
    // with two CTAs per SM still possible
    H.smem_sacc_off = schur / sizeof(double);
    H.schur_smem = 0;
    if (H.n_max > 0 && single_window && s + schur + (size_t)WARPS * H.blk * sizeof(double) <= 190 * 1024) {
        // mode 2 (default for a single window when it fits: reduced systems up to n = 48 with at most 195 keyframes in the
        // window's keyframe table): one private block per warp, one
        // CTA per SM.  Batches keep the RED path: there two CTAs per SM (different windows overlapping their latency-bound
        // phases) are worth more than the faster accumulation - measured 5.1 k vs 4.1 k solves/s on the C3 batch.
        H.schur_smem = 2;
        schur += (size_t)WARPS * H.blk * sizeof(double);
    } else if (H.n_max > 0 && H.n_max <= 96 && ncam <= MAX_CAMS) {
        // mode 3 (up to n = 96, single windows and batches): owner mode, see schur_owner_phase
        // Single windows spread over many CTAs stay on mode 2 when it fits (measured C3: 119 us vs 236 us per solve in the
        // Schur phase at 148 CTAs - there the phase is latency, not RED bound); batches (1-2 CTAs per window) take mode 3.
        // Its host-side pair sort counts over all ncam^2 keyframe pairs, so it is limited to windows of <= MAX_CAMS keyframes.
        const size_t R = (size_t)WARPS * (32 / H.sg);
        size_t tile = (R * (size_t)owner_tile_pitch(H.n_max) + 2 * R) * sizeof(double);
        const size_t stage = (size_t)WARPS * PCH * 26 * sizeof(double);
        if (tile < stage) tile = stage;
        H.schur_smem = 3;
        schur = (tile + 15) & ~(size_t)15;
    }
    // a keyframe table that does not fit next to the work area moves to the work block (balm_solve sizes it, one copy
    // per CTA of the group: every CTA writes its own candidate poses into it); the kernel code is the same either way
    const size_t work = (schur > solve ? schur : solve) + 16;
    H.cam_tab_global = s + work > SMEM_BUDGET;
    if (H.cam_tab_global) H.smem_work_off = 0;
    H.smem_bytes = H.cam_tab_global ? work : s + work;
    return OV2_OK;
}

static void fill_prob(const ov2_ba_problem* pb, const ov2_ba_opts* opts, const HostPlan& H, const Layout& L, Prob& P,
                      const double* Kh, const double* krh, const double* trlh, const int* stop_flag_dev) {
    memset(&P, 0, sizeof(P));
    P.ncam = pb->ncam; P.npts = pb->npts; P.nobs = pb->nobs;
    P.fx = Kh[0]; P.fy = Kh[1]; P.cx = Kh[2]; P.cy = Kh[3];
    P.rfx = P.fx; P.rfy = P.fy; P.rcx = P.cx; P.rcy = P.cy;
    for (int k = 0; k < 9; ++k) P.Rrl[k] = (k % 4 == 0) ? 1.0 : 0.0;
    if (pb->obs_type) {
        P.rfx = krh[0]; P.rfy = krh[1]; P.rcx = krh[2]; P.rcy = krh[3];
        const double qn = sqrt(trlh[3] * trlh[3] + trlh[4] * trlh[4] + trlh[5] * trlh[5] + trlh[6] * trlh[6]);
        const double x = trlh[3] / qn, y = trlh[4] / qn, z = trlh[5] / qn, w = trlh[6] / qn;
        const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                             2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                             2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
        for (int k = 0; k < 9; ++k) P.Rrl[k] = R[k];
        P.trl[0] = trlh[0]; P.trl[1] = trlh[1]; P.trl[2] = trlh[2];
    }
    P.th_f = (float)opts->huber_th;                       // const float mono_th (optimizer.cpp:47)
    P.huber_a = (double)sqrtf(P.th_f);                    // HuberLoss(std::sqrt(mono_th))
    P.huber_b = P.huber_a * P.huber_a;
    P.use_robust = opts->use_robust ? 1 : 0;
    P.apply_l2 = opts->apply_l2_after_robust ? 1 : 0;
    P.refine_loss = opts->refine_loss;
    P.max_it1 = opts->max_iters_robust; P.max_it2 = opts->max_iters_refine;
    P.ftol = opts->function_tolerance;
    P.stop_flag = stop_flag_dev;
    P.pose_const = (const uint8_t*)L.d(H.pc);
    P.lm_anchor_cam = (const int32_t*)L.d(H.lac);
    P.lm_anchor_px = (const double*)L.d(H.apx);
    P.obs_cam = (const int32_t*)L.d(H.oc);
    P.obs_lm = (const int32_t*)L.d(H.ol);
    P.obs_px = (const double*)L.d(H.opx);
    P.obs_type = pb->obs_type ? (const uint8_t*)L.d(H.ty) : nullptr;
    P.lm_ptr = (const int32_t*)L.d(H.lp);
    P.pose[0] = (double*)L.d(H.pose); P.pose[1] = (double*)L.d(H.pose1);
    P.invd[0] = (double*)L.d(H.invd); P.invd[1] = (double*)L.d(H.invd1);
    P.active = (uint8_t*)L.d(H.active); P.flags = (uint8_t*)L.d(H.flags);
    P.cam_used = (uint8_t*)L.d(H.camused); P.cam_slot = (int32_t*)L.d(H.camslot);
    P.Jr = (double*)L.d(H.Jr); P.Ja = (double*)L.d(H.Ja); P.Jo = (double*)L.d(H.Jo); P.Jl = (double*)L.d(H.Jl);
    P.chi2 = (double*)L.d(H.chi2); P.dpos = (uint8_t*)L.d(H.dpos);
    P.sc_lm = (double*)L.d(H.sclm); P.ete = (double*)L.d(H.ete); P.ge = (double*)L.d(H.ge);
    P.acc = (double*)L.d(H.acc); P.total = (double*)L.d(H.total); P.scal = (double*)L.d(H.scal);
    P.z = (double*)L.d(H.z); P.sc_cam = (double*)L.d(H.sccam); P.panel = (double*)L.d(H.panel);
    P.counts = (double*)L.d(H.counts); P.bar = (unsigned*)L.d(H.bar); P.result = (Result*)L.d(H.result);
    // OV2_BA_TRACE selects no path: it records per-phase times and prints the window's plan (read back by the plan tests)
    P.trace = getenv("OV2_BA_TRACE") ? (unsigned long long*)L.d(H.trace) : nullptr;
    P.ncv_max = H.ncv_max; P.blk = H.blk; P.solve_blocked = H.solve_blocked;
    P.sg = H.sg;   // lanes per landmark in the per-landmark phases
    P.cam_tab = H.cam_tab_global ? (double*)L.d(H.camtab) : nullptr;
    P.cam_tab_stride = H.tab_bytes / sizeof(double);
    P.schur_smem = H.schur_smem; P.smem_sacc_off = (int)H.smem_sacc_off;
    P.pair_perm = (const int32_t*)L.d(H.pp); P.pair_chunk = (const int2*)L.d(H.pch); P.npchunk = 0;
    P.smem_work_off = (int)H.smem_work_off;
}

// Solves `nprob` windows with one launch.  peers: multi-GPU exchange description (world 1 = none).
ov2_status balm_solve(ov2_ctx* ctx, int nprob, const ov2_ba_problem* pbs, const ov2_ba_opts* opts, ov2_ba_result* results,
                      uint8_t* const* outlier_outs, const Peers* peers, const int* stop_flag_dev) {
    if (!ctx || nprob <= 0 || !pbs || !opts || !results) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_localba_solve: bad arguments");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    const int world = peers ? peers->world : 1;
    std::vector<HostPlan> plans(nprob);
    std::vector<ov2_ba_problem> hp(nprob);           // host-resident views of every window (device inputs are copied down)
    std::vector<std::vector<char>> hold;              // storage for inputs that came as device pointers
    std::vector<Residence> where(nprob);
    Layout L;
    size_t smem_max = 0;
    int gmax_work = 1;
    for (int k = 0; k < nprob; ++k) {
        const ov2_ba_problem& pb = pbs[k];
        if (pb.ncam <= 0 || pb.npts < 0 || pb.nobs < 0 || (world == 1 && pb.npts <= 0))
            return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_localba_solve: bad arguments");
        hp[k] = pb;
        // the flattened window is host data in the reference's flow (optimizer.cpp:43-430); device-resident inputs are
        // accepted and staged through the host once (the solve itself never leaves the device)
        Residence& R = where[k];
        R.window = ov2_is_device_ptr(pb.pose);
        R.invd = R.on_device(pb.lm_invdepth);
        R.flags = R.on_device(outlier_outs ? outlier_outs[k] : nullptr);
        cudaError_t pull_err = cudaSuccess;
        auto pull = [&](const void* p, size_t bytes) -> const void* {
            if (!p || bytes == 0 || !R.on_device(p)) return p;
            hold.emplace_back(bytes);
            const cudaError_t ce = cudaMemcpy(hold.back().data(), p, bytes, cudaMemcpyDeviceToHost);
            if (ce != cudaSuccess) pull_err = ce;
            return hold.back().data();
        };
        hp[k].K = (const double*)pull(pb.K, 32);
        hp[k].pose_const = (const uint8_t*)pull(pb.pose_const, pb.ncam);
        hp[k].lm_anchor_cam = (const int32_t*)pull(pb.lm_anchor_cam, sizeof(int32_t) * (size_t)pb.npts);
        hp[k].lm_anchor_px = (const double*)pull(pb.lm_anchor_px, sizeof(double) * 2 * (size_t)pb.npts);
        hp[k].obs_cam = (const int32_t*)pull(pb.obs_cam, sizeof(int32_t) * (size_t)pb.nobs);
        hp[k].obs_lm = (const int32_t*)pull(pb.obs_lm, sizeof(int32_t) * (size_t)pb.nobs);
        hp[k].obs_px = (const double*)pull(pb.obs_px, sizeof(double) * 2 * (size_t)pb.nobs);
        hp[k].obs_type = (const uint8_t*)pull(pb.obs_type, (size_t)pb.nobs);
        hp[k].Kr = (const double*)pull(pb.Kr, 32);
        hp[k].Trl = (const double*)pull(pb.Trl, 56);
        if (pull_err != cudaSuccess) return ov2_fail(ctx, OV2_ERR_CUDA, "ov2_localba_solve: staging a device-resident window", pull_err);
        if (pb.obs_type && (!pb.Kr || !pb.Trl)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_localba_solve: obs_type given without Kr / Trl");
        if ((st = plan_window(ctx, &hp[k], world, L, plans[k], nprob == 1)) != OV2_OK) return st;
        if (plans[k].smem_bytes > smem_max) smem_max = plans[k].smem_bytes;
        const int wk = (pb.nobs + THREADS - 1) / THREADS;
        const int wl = (pb.npts + WARPS - 1) / WARPS;                  // a landmark per warp and phase (single window: every SM helps)
        const int w = wk > wl ? wk : wl;
        if (w > gmax_work) gmax_work = w;
    }
    if (smem_max > SMEM_BUDGET) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_localba_solve: window needs more than 200 KB of shared memory");
    // ---- launch geometry: G CTAs per window, all groups co-resident
    {
        // raised only when a window needs more than any before (a function-attribute change while another stream runs the
        // kernel may serialise with it)
        // (check + set + record under one lock: two host threads with their own contexts may make their first solves concurrently)
        static size_t attr_smem[16] = {0};
        static std::mutex attr_mu;
        std::lock_guard<std::mutex> attr_lock(attr_mu);
        const int dv = ctx->device & 15;
        if (smem_max > attr_smem[dv]) {
            OV2_CUDA(ctx, cudaFuncSetAttribute(ba_lm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
            attr_smem[dv] = smem_max;
        }
    }
    int per_sm = 0;
    OV2_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba_lm_kernel, THREADS, smem_max));
    if (per_sm < 1) return ov2_fail(ctx, OV2_ERR_CAPACITY, "ov2_localba_solve: kernel does not fit an SM");
    const int resident = per_sm * ctx->sm_count;
    int G = gmax_work < 1 ? 1 : gmax_work;
    // one wave of work per phase at most; more CTAs only add barrier latency
    int gcap = nprob == 1 ? resident : (resident / nprob < 1 ? 1 : resident / nprob);
    if (nprob > 1 && gcap > 16) gcap = 16;
    if (G > gcap) G = gcap;
    // OV2_BA_CTAS sets the group size within the cap: ranks that share one GPU need small groups to be co-resident, and
    // the group barrier and panel split are tested at chosen sizes.  Every size solves the same way.
    if (getenv("OV2_BA_CTAS")) { int e = atoi(getenv("OV2_BA_CTAS")); if (e >= 1 && e <= gcap) G = e; }
    if (world > 1 && G < 2) G = 2;
    int ngroups = nprob < resident / G ? nprob : resident / G;
    if (ngroups < 1) ngroups = 1;
    int grid = ngroups * G;
    // keyframe tables that live in the work block: one per CTA of the window's group
    for (int k = 0; k < nprob; ++k)
        if (plans[k].cam_tab_global) plans[k].camtab = L.take(RG_WORK, (size_t)G * plans[k].tab_bytes);
    // ---- pack the inputs into one pinned block: ONE H2D copy for the whole batch
    const size_t in_bytes = L.upload_bytes();
    const size_t host_need = in_bytes + L.bytes(RG_OUT);      // pinned: [packed inputs / returned states | returned output region]
    if (ctx->ba_ws_cap < host_need) {
        if (ctx->ba_ws) cudaFreeHost(ctx->ba_ws);
        ctx->ba_ws = nullptr; ctx->ba_ws_cap = 0;
        OV2_CUDA(ctx, cudaHostAlloc(&ctx->ba_ws, host_need * 2, cudaHostAllocDefault));
        ctx->ba_ws_cap = host_need * 2;
    }
    void *dup = nullptr, *dwork = nullptr;
    if ((st = ov2_scratch(ctx, in_bytes, &dup)) != OV2_OK) return st;
    if ((st = ov2_scratch(ctx, L.work_bytes() + 256, &dwork)) != OV2_OK) return st;
    L.place((char*)dup, (char*)dwork, (char*)ctx->ba_ws);
    // one window's share of the packing: validation, CSR by landmark, copies into the pinned block, the Prob record.
    // Windows write disjoint parts of the block, so a batch is packed by a few host threads.  Returns an error text.
    auto pack_window = [&](int k) -> const char* {
        const ov2_ba_problem& pb = hp[k];
        const HostPlan& H = plans[k];
        const int ncam = pb.ncam, npts = pb.npts, nobs = pb.nobs;
        // CSR by landmark (observations must be sorted by landmark)
        int32_t* lp = (int32_t*)L.h(H.lp);
        memset(lp, 0, sizeof(int32_t) * (size_t)(npts + 1));
        for (int i = 0; i < nobs; ++i) {
            const int l = pb.obs_lm[i];
            if (l < 0 || l >= npts || (i > 0 && l < pb.obs_lm[i - 1])) return "ov2_localba_solve: obs_lm must be sorted ascending and in range";
            lp[l + 1]++;
        }
        for (int l = 0; l < npts; ++l) lp[l + 1] += lp[l];
        for (int i = 0; i < nobs; ++i)
            if (pb.obs_cam[i] < 0 || pb.obs_cam[i] >= ncam) return "ov2_localba_solve: obs_cam out of range";
        for (int l = 0; l < npts; ++l)
            if (pb.lm_anchor_cam[l] < 0 || pb.lm_anchor_cam[l] >= ncam) return "ov2_localba_solve: lm_anchor_cam out of range";
        if (copy_state(L.h(H.pose), pbs[k].pose, sizeof(double) * 7 * ncam, where[k].window, cudaMemcpyDeviceToHost) != cudaSuccess)
            return "ov2_localba_solve: copying the poses failed";
        if (copy_state(L.h(H.invd), pbs[k].lm_invdepth, sizeof(double) * (size_t)npts, where[k].invd, cudaMemcpyDeviceToHost) != cudaSuccess)
            return "ov2_localba_solve: copying the inverse depths failed";
        memcpy(L.h(H.apx), pb.lm_anchor_px, sizeof(double) * 2 * (size_t)npts);
        memcpy(L.h(H.opx), pb.obs_px, sizeof(double) * 2 * (size_t)nobs);
        memcpy(L.h(H.lac), pb.lm_anchor_cam, sizeof(int32_t) * (size_t)npts);
        memcpy(L.h(H.oc), pb.obs_cam, sizeof(int32_t) * (size_t)nobs);
        memcpy(L.h(H.ol), pb.obs_lm, sizeof(int32_t) * (size_t)nobs);
        memcpy(L.h(H.pc), pb.pose_const, (size_t)ncam);
        if (pb.obs_type) memcpy(L.h(H.ty), pb.obs_type, (size_t)nobs);
        Prob P;
        fill_prob(&pb, opts, H, L, P, pb.K, pb.Kr, pb.Trl, stop_flag_dev);
        if (H.schur_smem == 3) {
            // stable counting sort of the observations by (anchor keyframe, observing keyframe), cut into chunks of <= PCH
            int32_t* perm = (int32_t*)L.h(H.pp);
            int2* chunks = (int2*)L.h(H.pch);
            std::vector<int32_t> head((size_t)ncam * ncam + 1, 0);
            for (int i = 0; i < nobs; ++i) head[(size_t)pb.lm_anchor_cam[pb.obs_lm[i]] * ncam + pb.obs_cam[i] + 1]++;
            for (size_t g = 0; g < (size_t)ncam * ncam; ++g) head[g + 1] += head[g];
            {
                std::vector<int32_t> cur(head.begin(), head.end() - 1);
                for (int i = 0; i < nobs; ++i) perm[cur[(size_t)pb.lm_anchor_cam[pb.obs_lm[i]] * ncam + pb.obs_cam[i]]++] = i;
            }
            int nch = 0;
            for (size_t g = 0; g < (size_t)ncam * ncam; ++g)
                for (int b = head[g]; b < head[g + 1]; b += PCH) {
                    if (nch >= H.pch_cap) return "ov2_localba_solve: pair chunk table overflow";
                    chunks[nch++] = make_int2(b, b + PCH < head[g + 1] ? b + PCH : head[g + 1]);
                }
            P.npchunk = nch;
        }
        memcpy(L.h(H.prob), &P, sizeof(P));
        return nullptr;
    };
    {
        int nthr = nprob >= 8 ? 8 : 1;
        const unsigned hc = std::thread::hardware_concurrency();
        if (hc > 0 && (unsigned)nthr > hc) nthr = (int)hc;
        std::atomic<int> next(0);
        std::atomic<const char*> perr(nullptr);
        auto worker = [&]() {
            for (int k = next.fetch_add(1); k < nprob; k = next.fetch_add(1)) {
                const char* e = pack_window(k);
                if (e) { perr.store(e); return; }
            }
        };
        if (nthr <= 1) worker();
        else {
            std::vector<std::thread> pool;
            for (int t = 1; t < nthr; ++t) pool.emplace_back(worker);
            worker();
            for (auto& t : pool) t.join();
        }
        if (perr.load()) return ov2_fail(ctx, OV2_ERR_INVALID, perr.load());
    }
    // the Prob records must be contiguous for the kernel: they are the first thing of each window's block, so gather them
    std::vector<Prob> parr(nprob);
    for (int k = 0; k < nprob; ++k) memcpy(&parr[k], L.h(plans[k].prob), sizeof(Prob));
    Prob* dprobs = nullptr;
    if ((st = ov2_scratch(ctx, (size_t)nprob, dprobs)) != OV2_OK) return st;
    cudaStream_t s = ctx->stream;
    OV2_CUDA(ctx, cudaMemcpyAsync(L.dev[RG_STATE], L.host[RG_STATE], in_bytes, cudaMemcpyHostToDevice, s));
    if (nprob == 1) dprobs = (Prob*)L.d(plans[0].prob);
    else OV2_CUDA(ctx, cudaMemcpyAsync(dprobs, parr.data(), sizeof(Prob) * (size_t)nprob, cudaMemcpyHostToDevice, s));   // parr outlives the sync below
    OV2_CUDA(ctx, cudaMemsetAsync(L.dev[RG_ZERO], 0, L.bytes(RG_ZERO) + L.bytes(RG_OUT), s));   // zero + output regions of every window
    OV2_CUDA(ctx, cudaMemsetAsync(L.dev[RG_ACT], 1, L.bytes(RG_ACT), s));                      // every observation starts active
    Peers X;
    memset(&X, 0, sizeof(X));
    X.world = 1;
    if (peers) X = *peers;
    const Prob* dp = dprobs;
    if (ctx->profiling) ov2_prof_begin(ctx);
    // grid <= resident capacity, so on a GPU this process owns every CTA starts at once.  A plain launch: cooperative
    // launches were measured to start their CTAs one after the other (~4 us each) and are not run concurrently with
    // another cooperative kernel (ranks sharing one GPU in the tests).  A CTA that never arrives trips the barrier timeout
    // instead of hanging the device.
    ba_lm_kernel<<<grid, THREADS, smem_max, s>>>(dp, nprob, G, X);
    const cudaError_t le = cudaGetLastError();
    ctx->launches++;
    if (le != cudaSuccess) return ov2_fail(ctx, OV2_ERR_CUDA, "ba_lm_kernel launch", le);
    if (ctx->profiling) ov2_prof_end(ctx, "ba_lm_kernel");
    // ---- results: [pose | invd] live in the input block (buffer 0), flags + result record in the work block
    OV2_CUDA(ctx, cudaMemcpyAsync(L.host[RG_STATE], L.dev[RG_STATE], L.bytes(RG_STATE), cudaMemcpyDeviceToHost, s));   // poses and inverse depths of every window: one copy
    OV2_CUDA(ctx, cudaMemcpyAsync(L.host[RG_OUT], L.dev[RG_OUT], L.bytes(RG_OUT), cudaMemcpyDeviceToHost, s));         // Result records + outlier flags: one copy
    auto wants_flags = [&](int k) { return outlier_outs && outlier_outs[k] && pbs[k].nobs > 0; };
    for (int k = 0; k < nprob; ++k)
        if (wants_flags(k) && where[k].flags)
            OV2_CUDA(ctx, cudaMemcpyAsync(outlier_outs[k], L.d(plans[k].flags), (size_t)pbs[k].nobs, cudaMemcpyDeviceToDevice, s));
    OV2_CUDA(ctx, cudaStreamSynchronize(s));
    std::vector<Result> hres(nprob);
    for (int k = 0; k < nprob; ++k) memcpy(&hres[k], L.h(plans[k].result), sizeof(Result));
    if (getenv("OV2_BA_TRACE")) {
        unsigned long long tr[16];
        cudaMemcpy(tr, L.d(plans[0].trace), sizeof(tr), cudaMemcpyDeviceToHost);
        static const char* names[16] = {"setup0", "A:eval", "B:schur", "B2:fold", "C:solve", "C:wait", "D:backsub", "E:ctl", "scan", "wb", "setup1", "bar0",
                                        "chol:P1", "chol:bar", "chol:P2", "chol:back|ownerB1"};
        fprintf(stderr, "[ba trace] G=%d grid=%d smem=%zu smemS=%d camtab=%s blocked=%d sg=%d |", G, grid, smem_max,
                plans[0].schur_smem, plans[0].cam_tab_global ? "global" : "shared", plans[0].solve_blocked, plans[0].sg);
        for (int k = 0; k < 16; ++k) fprintf(stderr, " %s %.1fus", names[k], tr[k] / 1e3);
        fprintf(stderr, "\n");
    }
    bool numeric_fail = false, aborted = false;
    for (int k = 0; k < nprob; ++k) {
        const HostPlan& H = plans[k];
        const size_t pb_bytes = sizeof(double) * 7 * pbs[k].ncam, ib = sizeof(double) * (size_t)pbs[k].npts;
        copy_state(pbs[k].pose, L.h(H.pose), pb_bytes, where[k].window, cudaMemcpyHostToDevice);
        copy_state(pbs[k].lm_invdepth, L.h(H.invd), ib, where[k].invd, cudaMemcpyHostToDevice);
        if (wants_flags(k) && !where[k].flags) memcpy(outlier_outs[k], L.h(H.flags), (size_t)pbs[k].nobs);
        ov2_ba_result& r = results[k];
        memset(&r, 0, sizeof(r));
        r.iters_robust = hres[k].iters_robust; r.iters_refine = hres[k].iters_refine;
        r.initial_cost = hres[k].initial_cost; r.final_cost = hres[k].final_cost;
        r.n_outliers_first = hres[k].n_outliers_first; r.n_outliers_second = hres[k].n_outliers_second;
        r.termination = hres[k].termination;
        if (r.termination == 2) numeric_fail = true;
        if (hres[k].aborted) aborted = true;
    }
    if (aborted) return ov2_fail(ctx, OV2_ERR_CUDA, "ov2_localba_solve: a barrier timed out (peer rank missing?)");
    if (numeric_fail) return ov2_fail(ctx, OV2_ERR_NUMERIC, "ov2_localba_solve: 5 consecutive invalid steps");
    return OV2_OK;
}
