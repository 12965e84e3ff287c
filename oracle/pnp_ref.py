"""CPU ORACLE for MultiViewGeometry::ceresPnP (motion-only BA).  TEST INFRASTRUCTURE ONLY.

"Next" row 2 of the scope table (SURVEY.md 8f): the pose refinement the front-end runs on every
frame right after KLT tracking (/root/reference/src/visual_front_end.cpp:783-801).  There is NO CUDA
implementation of this row yet - this module is step (a) of the row (oracle first); only tests/ may
import it.

numpy float64 restatement of /root/reference/src/multi_view_geometry.cpp:492-588:

  residual + analytic Jacobian   src/ceres_parametrization.cpp:300-356
                                 (DirectLeftSE3::ReprojectionErrorSE3::Evaluate: r = K (Tcw wpt) - unpx,
                                  d r / d xi = J_proj Rcw [-I | hat(wpt)] for the left perturbation
                                  T+ = exp(xi) T of SE3LeftParameterization)
  loss                           HuberLoss(sqrt(chi2th)) behind a LossFunctionWrapper (:507-512)
  solver                         Ceres 2.0 TrustRegionMinimizer + LevenbergMarquardtStrategy, DENSE_QR
                                 (:531-541): same loop as oracle/ba_ref.py::ceres_solve with a single
                                 6-dof block; the damped least-squares step is solved by a QR factorisation
                                 of [J; sqrt(D)] (dense_qr_solver.cc) - numpy.linalg.lstsq here
  two-stage flow                 outlier scan on the LAST Evaluate() of every block (chi2 > chi2th or
                                 depth <= 0, :552-566), all-outliers -> false (:568-570), optional second
                                 solve with the trivial loss on the inliers (:572-576)

Deliberately not modelled: options.max_solver_time_in_seconds = 0.005 (:538), a wall-clock cap that
makes the reference itself non-deterministic (Ceres checks it between iterations).

PINNING STATUS: pinned against the real Ceres 2.0 of the reference tree running the reference's own cost function with the calls
ceresPnP makes (DENSE_QR, Huber wrapper, outlier scan, L2 refinement): same outliers, verdict and pose to 1e-9
(tests/test_oracle_vs_reference_ceres.py::test_ceres_pnp_equals_real_ceres), and on the edge cases also termination, costs and
iteration count of every solve (::test_ceres_pnp_edges_and_iterations_equal_real_ceres; that build uses a stand-in linear-algebra header instead
of Eigen, see oracle/ba_ref.py).  Also: the Jacobian against central differences, the whole solve against ground truth and against
scipy.optimize.least_squares on the same cost (tests/test_oracle_pnp.py).
"""
from __future__ import annotations

import numpy as np

from .ba_ref import DBL_MAX, hat, huber, lm_step_accepted, lm_step_rejected, pose_plus, quat_normalize, quat_to_rot


def evaluate(pose, wpts, unpx, K, scales=None, need_jac=True):
    """ReprojectionErrorSE3::Evaluate for every block.  pose = Twc [t, q(xyzw)].
    Returns dict(r (n,2), chi2 (n,), depth_pos (n,), J (n,2,6) or None)."""
    fx, fy, cx, cy = (float(v) for v in K)
    t, q = pose[:3], quat_normalize(pose[3:])
    Rwc = quat_to_rot(q)
    Rcw = Rwc.T
    pc = (wpts - t) @ Rcw.T                       # Tcw * wpt
    invz = 1.0 / pc[:, 2]
    pred = np.stack([fx * pc[:, 0] * invz + cx, fy * pc[:, 1] * invz + cy], 1)
    sinfo = np.ones(len(wpts)) if scales is None else 1.0 / np.power(2.0, np.asarray(scales, np.float64))
    r = (pred - unpx) * sinfo[:, None]
    out = dict(r=r, chi2=(r ** 2).sum(1), depth_pos=pc[:, 2] > 0, J=None)
    if need_jac:
        invz2 = invz * invz
        Jcam = np.zeros((len(wpts), 2, 3))
        Jcam[:, 0, 0] = invz * fx
        Jcam[:, 0, 2] = -pc[:, 0] * invz2 * fx
        Jcam[:, 1, 1] = invz * fy
        Jcam[:, 1, 2] = -pc[:, 1] * invz2 * fy
        JR = Jcam @ Rcw                           # (n,2,3)
        J = np.zeros((len(wpts), 2, 6))
        J[:, :, :3] = -JR
        J[:, :, 3:] = np.einsum("nij,njk->nik", JR, np.stack([hat(w) for w in wpts]))
        out["J"] = J * sinfo[:, None, None]
    return out


def ceres_solve_pose(pose, wpts, unpx, K, active, max_iters, huber_a, scales=None, function_tolerance=1e-3, log=None):
    """ceres::Solve on the residual blocks `active` with one SE3 block, DENSE_QR, Ceres 2.0 defaults
    (jacobi scaling, initial radius 1e4, eta irrelevant for a direct solver).  Returns
    (pose, summary, last) with last = chi2 / depth_pos of the last Evaluate() of each active block.

    summary["stop"] names the test that ended the solve: "max_iterations", "gradient" and "radius" are checked at the top of
    the loop (Ceres' FinalizeIterationAndCheckIfMinimizerCanContinue, after it has recorded the iteration), "parameter",
    "function" and "invalid" inside an iteration (Ceres returns before recording it).  So Ceres' Summary::iterations.size(),
    which counts iteration 0, is summary["iterations"] + 1 for the first three and summary["iterations"] for the others.

    log: when a list, one entry per decision the loop takes, with the values each decision compares:
      {"gmax"}                                      gradient max-norm of an accepted point (against 1e-10)
      {"it", "valid", "radius"}                     a step the linear solve could not use
      {"it", "step_norm", "xnorm", "x_cost", "cand_cost", "mcc", "rho", "radius"}
                                                    a valid step: step norm against 1e-8 (xnorm + 1e-8), |x_cost - cand_cost|
                                                    against function_tolerance x_cost, rho against 1e-3 (rho is None when a
                                                    tolerance ended the solve first)"""
    pose = np.asarray(pose, np.float64).copy()
    idx = np.nonzero(active)[0]
    last = dict(chi2=np.zeros(len(active)), depth_pos=np.ones(len(active), bool))
    summ = dict(iterations=0, termination="NO_CONVERGENCE", stop="max_iterations", initial_cost=0.0, final_cost=0.0, usable=True)
    if len(idx) == 0:
        summ["termination"], summ["stop"] = "CONVERGENCE", "no_blocks"
        return pose, summ, last
    W, U = wpts[idx], unpx[idx]
    sc = None if scales is None else np.asarray(scales)[idx]

    def record(ev):
        last["chi2"][idx] = ev["chi2"]
        last["depth_pos"][idx] = ev["depth_pos"]

    def cost_and_w(ev):
        s = ev["chi2"]
        if huber_a is None:
            return 0.5 * s.sum(), np.ones_like(s)
        rho = huber(s, huber_a)
        return 0.5 * rho[0].sum(), np.sqrt(rho[1])          # rho'' <= 0: the corrector only rescales

    def eval_jac(p):
        ev = evaluate(p, W, U, K, sc, True)
        record(ev)
        cost, w = cost_and_w(ev)
        return cost, (ev["r"] * w[:, None]).reshape(-1), (ev["J"] * w[:, None, None]).reshape(-1, 6)

    x_cost, r, J = eval_jac(pose)
    scale = 1.0 / (1.0 + np.sqrt((J ** 2).sum(0)))         # jacobi scaling, computed once
    g = J.T @ r
    gmax = np.abs(np.concatenate([pose[:3], quat_normalize(pose[3:])]) - pose_plus(pose, -g)).max()
    J = J * scale
    if log is not None:
        log.append(dict(gmax=gmax))
    summ["initial_cost"] = x_cost
    minimum_cost, best = DBL_MAX, pose.copy()
    xnorm = -1.0
    radius, decrease_factor, reuse_diag, diag = 1e4, 2.0, False, None
    step_successful, num_invalid, iteration = True, 0, 0
    while True:
        if step_successful and x_cost < minimum_cost:
            minimum_cost, best = x_cost, pose.copy()
        if iteration >= max_iters:
            break
        if step_successful and gmax <= 1e-10:
            summ["termination"], summ["stop"] = "CONVERGENCE", "gradient"
            break
        if radius <= 1e-32:
            summ["termination"], summ["stop"] = "CONVERGENCE", "radius"
            break
        iteration += 1
        if not reuse_diag:
            diag = np.clip((J ** 2).sum(0), 1e-6, 1e32)
        D = np.sqrt(diag / radius)
        reuse_diag = True
        A = np.vstack([J, np.diag(D)])
        b = np.concatenate([-r, np.zeros(6)])
        step, *_ = np.linalg.lstsq(A, b, rcond=None)       # DENSE_QR on the augmented system
        Jstep = J @ step
        model_cost_change = -(Jstep * (r + Jstep / 2.0)).sum()
        if not (np.isfinite(step).all() and model_cost_change > 0.0):
            if log is not None:
                log.append(dict(it=iteration, valid=False, radius=radius))
            num_invalid += 1
            if num_invalid >= 5:
                summ["termination"], summ["stop"] = "FAILURE", "invalid"
                summ["usable"] = False
                break
            radius, decrease_factor = lm_step_rejected(radius, decrease_factor)
            step_successful = False
            continue
        num_invalid = 0
        cand = pose_plus(pose, step * scale)
        ev = evaluate(cand, W, U, K, sc, False)
        record(ev)
        cand_cost, _ = cost_and_w(ev)
        if not np.isfinite(cand_cost):
            cand_cost = DBL_MAX
        step_norm = np.sqrt(((pose - cand) ** 2).sum())
        entry = dict(it=iteration, valid=True, step_norm=step_norm, xnorm=xnorm, x_cost=x_cost, cand_cost=cand_cost, mcc=model_cost_change,
                     rho=None, radius=radius)
        if log is not None:
            log.append(entry)
        if step_norm <= 1e-8 * (xnorm + 1e-8):
            summ["termination"], summ["stop"] = "CONVERGENCE", "parameter"
            break
        if abs(x_cost - cand_cost) <= function_tolerance * x_cost:
            summ["termination"], summ["stop"] = "CONVERGENCE", "function"
            break
        rel = -DBL_MAX if cand_cost >= DBL_MAX else (x_cost - cand_cost) / model_cost_change
        entry["rho"] = rel
        if rel > 1e-3:
            pose = cand
            xnorm = np.sqrt((pose ** 2).sum())
            x_cost, r, J = eval_jac(pose)
            g = J.T @ r
            gmax = np.abs(pose - pose_plus(pose, -g)).max()
            J = J * scale
            if log is not None:
                log.append(dict(gmax=gmax))
            step_successful = True
            radius = lm_step_accepted(radius, rel)
            decrease_factor, reuse_diag = 2.0, False
        else:
            step_successful = False
            radius, decrease_factor = lm_step_rejected(radius, decrease_factor)
    summ["iterations"] = iteration
    summ["final_cost"] = minimum_cost if minimum_cost < DBL_MAX else x_cost
    return best, summ, last


def ceres_pnp(unpx, wpts, Twc, K, nmaxiter=5, chi2th=5.9915, use_robust=True, apply_l2_after_robust=True, scales=None, summary=False):
    """MultiViewGeometry::ceresPnP.  Returns (success, Twc_out, outlier indices); with summary=True also a dict:
    summary      the Solver::Summary of the last solve that ran (see ceres_solve_pose)
    solves       the summaries of every solve that ran (1 or 2)
    log          per solve, the decision log of ceres_solve_pose
    chi2, depth_pos, chi2th
                 what the outlier scan after the first solve compared: chi2 > chi2th or not depth_pos is an outlier."""
    unpx = np.asarray(unpx, np.float64).reshape(-1, 2)
    wpts = np.asarray(wpts, np.float64).reshape(-1, 3)
    n = len(unpx)
    active = np.ones(n, bool)
    a = float(np.sqrt(np.float32(chi2th))) if use_robust else None     # chi2th is a float argument (:496)
    chi2th = float(np.float32(chi2th))
    logs = [[]]
    pose, summ, last = ceres_solve_pose(np.asarray(Twc, np.float64), wpts, unpx, K, active, nmaxiter, a, scales, log=logs[0])
    info = dict(summary=summ, solves=[summ], log=logs, chi2=last["chi2"].copy(), depth_pos=last["depth_pos"].copy(), chi2th=chi2th)
    bad = (last["chi2"] > chi2th) | ~last["depth_pos"]
    outliers = np.nonzero(bad)[0]
    if len(outliers) == n:
        ret = (False, np.asarray(Twc, np.float64).copy(), outliers)   # Twc is not written back (:568-570)
        return ret + (info,) if summary else ret
    if apply_l2_after_robust and len(outliers):
        logs.append([])
        pose, summ, last = ceres_solve_pose(pose, wpts, unpx, K, ~bad, nmaxiter, None, scales, log=logs[1])
        info["summary"] = summ
        info["solves"].append(summ)
    ret = (bool(summ["usable"]), pose, outliers)
    return ret + (info,) if summary else ret
