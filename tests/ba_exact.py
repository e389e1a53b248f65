"""Float64 restatement of the landmark bundle adjustment (`csrc/landmark_ba.cu`, `rgbdslam_b200_landmark_ba`) -- TEST INFRASTRUCTURE.

Written from g2o's formulas, vectorised, not from the kernels:
- `linearize`: EdgeSE3PointXYZDepth error and analytic Jacobians per observation (blocks Hcc, Hcp, Hpp, bc, bp with
  H = J'WJ, b = -J'We), the EdgeSE3 error and Jacobians of the C oracle (`oracle.edge_se3`) with the Huber weight rho'(e'We).
- `chi2`: plain observation chi2 plus robust pose-edge chi2, summed with math.fsum.
- `trial`: one damped step with the points eliminated -- per-point (Hpp + lambda I)^-1, the reduced camera system S dc = g formed
  densely, block-Jacobi PCG with the solver's stop rule, a direct solve of the same system, back-substitution, VertexSE3::oplus
  (`oracle.vertex_oplus`), the LM scale.
- `optimize`: the Levenberg-Marquardt bookkeeping of `lm_optimize` (csrc/posegraph.h), every trial recorded.
- `make_ba_corridor`: cameras along a corridor, each seeing a sliding window of landmarks, with the topology options that reach
  the kernels' CTA, warp and block boundaries.
"""
from __future__ import annotations

import math
import sys

import numpy as np
import scipy.sparse as sp

from oracle import oracle as co

PCG_REL_TOL = 1e-18   # r'M^-1 r <= 1e-18 r0'M^-1 r0 (ba_cg_step_kernel's rel_tol)
PCG_BURST = 16        # the host checks the PCG state after every 16 steps
CERT_BAND = 1e-6      # a PCG stop is certified when dn/dn0 lies outside 1e-18 * [1 - band, 1 + band] at the stop and before
RHO_BAND = 1e-6       # an LM decision is certified when |rho| > band ...
CHI2_BAND = 1e-9      # ... and the trial chi2 differs from the current one by more than this, relative
DBL_MAX = sys.float_info.max


# ---- geometry -----------------------------------------------------------------------------------------------------
def rot(q):
    """rotation matrices of (..., 4) quaternions (x, y, z, w), normalised first"""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - z * w); R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w); R[..., 2, 1] = 2 * (y * z + x * w); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def obs_terms(poses, points, oc, op, uvd, K4, jac=True):
    """EdgeSE3PointXYZDepth per observation: error e (n, 3) in the form (fx x + cx z) / z - u, and with `jac` the Jacobians
    Jc (n, 3, 6) w.r.t. the right-multiplicative camera increment (t, qx, qy, qz) and Jp (n, 3, 3) w.r.t. the point."""
    fx, fy, cx, cy = (float(v) for v in K4)
    R = rot(poses[oc, 3:])
    zc = np.einsum("nji,nj->ni", R, points[op] - poses[oc, :3])   # R'(p - t)
    x, y, z = zc[:, 0], zc[:, 1], zc[:, 2]
    zp0, zp1 = fx * x + cx * z, fy * y + cy * z
    e = np.stack([zp0 / z - uvd[:, 0], zp1 / z - uvd[:, 1], z - uvd[:, 2]], 1)
    if not jac:
        return e
    n = len(oc)
    Jz = np.zeros((n, 3, 9))                  # d zc / d (dt, dq, p): [-I | 2 [zc]x | R']
    Jz[:, 0, 0] = Jz[:, 1, 1] = Jz[:, 2, 2] = -1.0
    Jz[:, 0, 4], Jz[:, 0, 5] = -2 * z, 2 * y
    Jz[:, 1, 3], Jz[:, 1, 5] = 2 * z, -2 * x
    Jz[:, 2, 3], Jz[:, 2, 4] = -2 * y, 2 * x
    Jz[:, :, 6:] = np.transpose(R, (0, 2, 1))
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    dzp = np.einsum("ab,nbk->nak", K, Jz)
    J = np.empty_like(Jz)
    J[:, 0] = (dzp[:, 0] * z[:, None] - zp0[:, None] * dzp[:, 2]) / (z * z)[:, None]
    J[:, 1] = (dzp[:, 1] * z[:, None] - zp1[:, None] * dzp[:, 2]) / (z * z)[:, None]
    J[:, 2] = dzp[:, 2]
    return e, J[:, :, :6], J[:, :, 6:]


def oplus(pose, d):
    """VertexSE3::oplus through the C oracle"""
    return co.vertex_oplus(pose, d)


# ---- the problem --------------------------------------------------------------------------------------------------
class Problem:
    """One landmark_ba input (the arrays of rgbdslam_b200_landmark_ba), poses (nc, 7) world-from-camera (t, q)."""

    def __init__(self, poses, fixed, points, obs_cam, obs_point, obs_uvd, obs_info3, K4, ij=None, meas=None, info=None,
                 huber_delta=1.0):
        self.poses = np.array(poses, np.float64).reshape(-1, 7)
        self.fixed = np.asarray(fixed).astype(bool)
        self.points = np.array(points, np.float64).reshape(-1, 3)
        self.oc, self.op = np.asarray(obs_cam, np.int64), np.asarray(obs_point, np.int64)
        self.uvd = np.asarray(obs_uvd, np.float64).reshape(-1, 3)
        self.w3 = np.asarray(obs_info3, np.float64).reshape(-1, 3)
        self.K4 = np.asarray(K4, np.float64)
        self.ij = np.zeros((0, 2), np.int64) if ij is None else np.asarray(ij, np.int64).reshape(-1, 2)
        self.meas = np.zeros((0, 7)) if meas is None else np.asarray(meas, np.float64).reshape(-1, 7)
        self.info = np.zeros((0, 36)) if info is None else np.asarray(info, np.float64).reshape(-1, 36)
        self.delta = float(huber_delta)
        self.nc, self.np_ = len(self.poses), len(self.points)
        # the observation incidence, both ways (CSR order does not matter to the algebra)
        self.B_rows = None

    @classmethod
    def from_dict(cls, d, edges=True, huber_delta=1.0):
        kw = dict(ij=d["ij"], meas=d["meas"], info=d["info"]) if edges and "ij" in d else {}
        return cls(d["poses"], d["fixed"], d["points"], d["obs_cam"], d["obs_point"], d["obs_uvd"], d["obs_info3"], d["K4"],
                   huber_delta=huber_delta, **kw)

    def with_state(self, poses, points):
        q = object.__new__(Problem)
        q.__dict__.update(self.__dict__)
        q.poses, q.points = np.array(poses, np.float64), np.array(points, np.float64)
        return q

    # ---- chi2 ----
    def edge_terms(self, poses, jac=True):
        """per pose edge: (e, Ji, Jj, e'We, rho') with rho' the Huber weight"""
        out = []
        for k, (i, j) in enumerate(self.ij):
            e, Ji, Jj = co.edge_se3(poses[i], poses[j], self.meas[k], want_jac=jac)
            W = self.info[k].reshape(6, 6)
            e2 = float(e @ W @ e)
            w = 1.0 if e2 <= self.delta ** 2 else self.delta / math.sqrt(e2)
            out.append((e, Ji, Jj, e2, w))
        return out

    def chi2_terms(self, poses=None, points=None):
        poses = self.poses if poses is None else poses
        points = self.points if points is None else points
        terms = []
        if len(self.oc):
            e = obs_terms(poses, points, self.oc, self.op, self.uvd, self.K4, jac=False)
            terms.extend((e * e * self.w3).sum(1).tolist())
        d2 = self.delta ** 2
        for _, _, _, e2, _ in self.edge_terms(poses, jac=False):
            terms.append(e2 if e2 <= d2 else 2 * math.sqrt(e2) * self.delta - d2)
        return terms

    def chi2(self, poses=None, points=None):
        """plain observation chi2 + robust (Huber) pose-edge chi2, math.fsum"""
        return math.fsum(self.chi2_terms(poses, points))

    # ---- normal equations ----
    def linearize(self):
        """per-observation blocks and per-camera pose-edge sums at the current state"""
        nc = self.nc
        L = {}
        if len(self.oc):
            e, Jc, Jp = obs_terms(self.poses, self.points, self.oc, self.op, self.uvd, self.K4)
            W = self.w3
            L["Hcc"] = np.einsum("nri,nr,nrj->nij", Jc, W, Jc)
            L["Hcp"] = np.einsum("nri,nr,nrj->nij", Jc, W, Jp)
            L["Hpp"] = np.einsum("nri,nr,nrj->nij", Jp, W, Jp)
            L["bc"] = -np.einsum("nri,nr,nr->ni", Jc, W, e)
            L["bp"] = -np.einsum("nri,nr,nr->ni", Jp, W, e)
        else:
            L.update(Hcc=np.zeros((0, 6, 6)), Hcp=np.zeros((0, 6, 3)), Hpp=np.zeros((0, 3, 3)), bc=np.zeros((0, 6)),
                     bp=np.zeros((0, 3)))
        Hcam = np.zeros((nc, 6, 6)); bcam = np.zeros((nc, 6))
        np.add.at(Hcam, self.oc, L["Hcc"]); np.add.at(bcam, self.oc, L["bc"])
        off = []                                   # (i, j, C) with C = w Ji'W Jj
        for k, (e, Ji, Jj, e2, w) in enumerate(self.edge_terms(self.poses)):
            i, j = self.ij[k]
            W = self.info[k].reshape(6, 6)
            Hcam[i] += w * Ji.T @ W @ Ji
            Hcam[j] += w * Jj.T @ W @ Jj
            bcam[i] -= w * Ji.T @ W @ e
            bcam[j] -= w * Jj.T @ W @ e
            if i != j:
                off.append((i, j, w * Ji.T @ W @ Jj))
        L["Hcam"], L["bcam"], L["off"] = Hcam, bcam, off
        Hp = np.zeros((self.np_, 3, 3)); bp = np.zeros((self.np_, 3)); cnt = np.zeros(self.np_, np.int64)
        np.add.at(Hp, self.op, L["Hpp"]); np.add.at(bp, self.op, L["bp"]); np.add.at(cnt, self.op, 1)
        L["Hp"], L["bpt"], L["cnt"] = Hp, bp, cnt
        return L

    def max_diag(self, L):
        """computeLambdaInit's max diag(H) at lambda = 0 over the free cameras and all points"""
        m = 0.0
        free = ~self.fixed
        if free.any():
            m = max(m, float(np.diagonal(L["Hcam"][free], axis1=1, axis2=2).max()))
        if self.np_:
            m = max(m, float(np.diagonal(L["Hp"], axis1=1, axis2=2).max()))
        return m

    def full_system(self, L, lam):
        """the un-eliminated damped system (6 nc + 3 np) with the fixed cameras' rows and columns dropped: (A, b, free mask)"""
        nc, npt = self.nc, self.np_
        n = 6 * nc + 3 * npt
        H = np.zeros((n, n)); b = np.zeros(n)
        for c in range(nc):
            H[6 * c:6 * c + 6, 6 * c:6 * c + 6] += L["Hcam"][c]
            b[6 * c:6 * c + 6] += L["bcam"][c]
        for i, j, C in L["off"]:
            H[6 * i:6 * i + 6, 6 * j:6 * j + 6] += C
            H[6 * j:6 * j + 6, 6 * i:6 * i + 6] += C.T
        for o in range(len(self.oc)):
            c, p = self.oc[o], 6 * nc + 3 * self.op[o]
            H[6 * c:6 * c + 6, p:p + 3] += L["Hcp"][o]
            H[p:p + 3, 6 * c:6 * c + 6] += L["Hcp"][o].T
        for q in range(npt):
            H[6 * nc + 3 * q:6 * nc + 3 * q + 3, 6 * nc + 3 * q:6 * nc + 3 * q + 3] += L["Hp"][q]
            b[6 * nc + 3 * q:6 * nc + 3 * q + 3] += L["bpt"][q]
        free = np.ones(n, bool)
        for c in np.nonzero(self.fixed)[0]:
            free[6 * c:6 * c + 6] = False
        return H + lam * np.eye(n), b, free

    def reduced(self, L, lam):
        """the points eliminated at damping lam: Hpp^-1, bp, S (dense, free cameras), g, the block-Jacobi preconditioner"""
        nc, npt = self.nc, self.np_
        I3, I6 = np.eye(3), np.eye(6)
        Hd = L["Hp"] + lam * I3
        ok = (L["cnt"] > 0) & (np.linalg.det(Hd) > 0)     # a point without observations drops out of the system
        Hinv = np.zeros_like(Hd)
        if ok.any():
            Hinv[ok] = np.linalg.inv(Hd[ok])
        bp = np.where(ok[:, None], L["bpt"], 0.0)
        Hcc = L["Hcam"] + lam * I6
        # the sparse coupling Hcp (6 nc x 3 np), duplicate (camera, point) observations summed
        no = len(self.oc)
        rows = (6 * self.oc[:, None, None] + np.arange(6)[None, :, None]).repeat(3, 2)
        cols = (3 * self.op[:, None, None] + np.arange(3)[None, None, :]).repeat(6, 1)
        B = sp.csr_matrix((L["Hcp"].reshape(-1), (rows.reshape(-1), cols.reshape(-1))), shape=(6 * nc, 3 * npt)) if no else \
            sp.csr_matrix((6 * nc, 3 * npt))
        hr = (3 * np.arange(npt)[:, None, None] + np.arange(3)[None, :, None]).repeat(3, 2)
        Hi = sp.csr_matrix((Hinv.reshape(-1), (hr.reshape(-1), np.transpose(hr, (0, 2, 1)).reshape(-1))), shape=(3 * npt, 3 * npt))
        S = np.zeros((6 * nc, 6 * nc))
        for c in range(nc):
            S[6 * c:6 * c + 6, 6 * c:6 * c + 6] = Hcc[c]
        for i, j, C in L["off"]:
            S[6 * i:6 * i + 6, 6 * j:6 * j + 6] += C
            S[6 * j:6 * j + 6, 6 * i:6 * i + 6] += C.T
        if no and npt:
            S -= (B @ Hi @ B.T).toarray()
        g = L["bcam"].reshape(-1) - (B @ (Hi @ bp.reshape(-1)) if no and npt else 0.0)
        # preconditioner: the inverse of Hcc - sum over the camera's observations of Hcp_o Hpp^-1 Hpc_o, one term per
        # observation (as ba_cams_kernel sums it: with duplicate (camera, point) observations this is not exactly S's diagonal
        # block; any SPD block-Jacobi matrix gives the same PCG solution)
        Mb = Hcc.copy()
        if no:
            Y = np.einsum("nij,njk->nik", L["Hcp"], Hinv[self.op])
            np.add.at(Mb, self.oc, -np.einsum("nik,njk->nij", Y, L["Hcp"]))
        free = ~self.fixed
        Minv = np.zeros_like(Mb)
        if free.any():
            Minv[free] = np.linalg.inv(Mb[free])
        fm = np.repeat(free, 6)
        g = np.where(fm, g, 0.0)
        # magnitudes of the summands behind g and S (for the rounding floor of step_bound): sum |terms| per entry
        gabs = np.zeros((nc, 6)); np.add.at(gabs, self.oc, np.abs(L["bc"]))
        for k, (e, Ji, Jj, e2, w) in enumerate(self.edge_terms(self.poses)) if len(self.ij) else ():
            W = self.info[k].reshape(6, 6)
            gabs[self.ij[k, 0]] += np.abs(w * Ji.T @ W @ e); gabs[self.ij[k, 1]] += np.abs(w * Jj.T @ W @ e)
        gabs = gabs.reshape(-1)
        Sabs = np.abs(S)
        if no and npt:
            Ba, Ha = abs(B), abs(Hi)
            gabs = gabs + Ba @ (Ha @ np.abs(bp).reshape(-1))
            Sabs = Sabs + (Ba @ Ha @ Ba.T).toarray()
        nterms = np.bincount(self.oc, minlength=nc) + (np.bincount(self.ij.reshape(-1), minlength=nc) if len(self.ij) else 0)
        return dict(Hinv=Hinv, bp=bp, S=S, g=g, Minv=Minv, free=fm, B=B, bc=np.where(fm, L["bcam"].reshape(-1), 0.0),
                    gabs=gabs, Sabs=Sabs, nterms=int(nterms.max(initial=0)), ptterms=int(L["cnt"].max(initial=0)))

    def rounding_floor(self, R, xc):
        """How far two float64 evaluations of the same step may differ through rounding alone, (camera, point) max norm.
        Every entry of g and S is a sum of at most n terms (observations and pose-edge incidences of a camera) each carrying a
        few roundings of its own: summed in another order it may move by (n + 8) eps sum |terms|.  That perturbs the
        solution by at most |S^-1| (dg + dS |x|) entrywise, and the back-substitution carries it into the points."""
        f = R["free"]
        eps = np.finfo(np.float64).eps
        dc = np.zeros(len(xc))
        if f.any():
            Si = np.abs(np.linalg.inv(R["S"][np.ix_(f, f)]))
            dc[f] = (R["nterms"] + 8) * eps * (Si @ (R["gabs"][f] + R["Sabs"][np.ix_(f, f)] @ np.abs(xc[f])))
        if not self.np_:
            return float(dc.max(initial=0.0)), 0.0
        Ha = np.abs(R["Hinv"])
        t = np.abs(R["bp"]).reshape(-1) + (abs(R["B"]).T @ np.abs(xc) if len(self.oc) else 0.0)
        tp = (R["ptterms"] + 8) * eps * t + (abs(R["B"]).T @ dc if len(self.oc) else 0.0)
        dp = np.einsum("pij,pj->pi", Ha, tp.reshape(-1, 3))
        return float(dc.max(initial=0.0)), float(dp.max(initial=0.0))

    def back_substitute(self, R, xc):
        """dp = Hpp^-1 (bp - Hpc dc)"""
        if not self.np_:
            return np.zeros((0, 3))
        t = R["bp"].reshape(-1) - (R["B"].T @ xc if len(self.oc) else 0.0)
        return np.einsum("pij,pj->pi", R["Hinv"], t.reshape(-1, 3))

    def apply(self, xc, dp):
        poses = self.poses.copy()
        for c in np.nonzero(~self.fixed)[0]:
            poses[c] = oplus(self.poses[c], xc[6 * c:6 * c + 6])
        return poses, self.points + dp


def pcg(S, g, Minv, free, n_cams):
    """block-Jacobi PCG on S x = g over the free rows (x = 0 on the fixed cameras), the solver's stop rule and iteration cap.
    Returns (x, iterations, status, ratios) with status 'converged' / 'cap' / 'breakdown' and ratios the dn / dn0 sequence."""
    f = free
    A, b = S[np.ix_(f, f)], g[f]
    nb = int(f.sum()) // 6
    M = np.zeros((int(f.sum()), int(f.sum())))
    for k, c in enumerate(np.nonzero(f[::6])[0]):
        M[6 * k:6 * k + 6, 6 * k:6 * k + 6] = Minv[c]
    cap = -(-(6 * n_cams + 20) // PCG_BURST) * PCG_BURST
    x = np.zeros_like(b)
    r = b.copy()
    s = M @ r
    d = s.copy()
    dn = float(r @ s)
    dn0 = dn
    ratios = [1.0]
    it, status = 0, "converged" if dn0 <= 0 else "cap"
    while status == "cap" and it < cap:
        q = A @ d
        dq = float(d @ q)
        if not dq > 0:
            status = "breakdown"
            break
        alpha = dn / dq
        x += alpha * d
        r -= alpha * q
        s = M @ r
        dn_new = float(r @ s)
        d = s + (dn_new / dn) * d
        dn = dn_new
        it += 1
        ratios.append(dn / dn0)
        if dn <= dn0 * PCG_REL_TOL:
            status = "converged"
    out = np.zeros_like(g)
    out[f] = x
    return out, it, status, ratios


def pcg_certified(it, status, ratios):
    """the stop index is certain: converged (not capped, not broken down) with dn/dn0 outside 1e-18 (1 +- band) at the stop
    and at the index before it"""
    if status != "converged":
        return False
    if it == 0:
        return True
    lo, hi = PCG_REL_TOL * (1 - CERT_BAND), PCG_REL_TOL * (1 + CERT_BAND)
    return ratios[it] < lo and ratios[it - 1] > hi


def trial(P: Problem, L, lam):
    """one damped step: the PCG step and the direct step of the same reduced system, the trial state and its chi2"""
    R = P.reduced(L, lam)
    xc, it, status, ratios = pcg(R["S"], R["g"], R["Minv"], R["free"], P.nc)
    f = R["free"]
    x_dir = np.zeros_like(R["g"])
    if f.any():
        x_dir[f] = np.linalg.solve(R["S"][np.ix_(f, f)], R["g"][f])
    dp = P.back_substitute(R, xc)
    dp_dir = P.back_substitute(R, x_dir)
    scale = math.fsum((dp * (lam * dp + R["bp"])).reshape(-1).tolist() + (xc * (lam * xc + R["bc"])).tolist())
    poses, points = P.apply(xc, dp)
    ok = status != "breakdown"
    temp = P.chi2(poses, points)
    floor = P.rounding_floor(R, xc)
    return dict(lam=lam, xc=xc, dp=dp, xc_dir=x_dir, dp_dir=dp_dir, floor_c=floor[0], floor_p=floor[1],
                pcg_iterations=it, pcg_status=status, ratios=ratios,
                pcg_certified=pcg_certified(it, status, ratios), ok=ok, temp=temp if ok else DBL_MAX, temp_eval=temp,
                scale=scale, poses=poses, points=points)


def step_bound(t):
    """How far a GPU step may lie from the restatement's PCG step in the max norm, for cameras and points.
    Both PCGs run the same recurrence to the same stopping index; each iterate lies within |x_pcg - x_direct| of the exact
    solution up to that iterate's own rounding, so the two iterates lie within 2 |x_pcg - x_direct| of each other; the
    residual the stop admits and the float64 rounding of two different summation orders (kernel CSR order against numpy's)
    at most double that again, and the final factor 2 covers the Krylov sequences drifting apart by one rounding-level step
    over hundreds of iterations.  The 1e-12 |step| term is the float64 rounding of the PCG recurrences themselves when the
    PCG error is below it.  Near the optimum g is a small difference of large sums and its rounding, not the PCG, decides how
    far two evaluations of the step may lie apart: Problem.rounding_floor bounds that part, and it is added as it is."""
    bc = 8 * np.abs(t["xc"] - t["xc_dir"]).max(initial=0.0) + 1e-12 * np.abs(t["xc"]).max(initial=0.0) + t["floor_c"]
    bp = 8 * np.abs(t["dp"] - t["dp_dir"]).max(initial=0.0) + 1e-12 * np.abs(t["dp"]).max(initial=0.0) + t["floor_p"]
    return bc, bp


def optimize(P: Problem, iterations):
    """lm_optimize (csrc/posegraph.h) on the restatement.  Returns dict(poses, points, chi2_before, chi2, lm_iterations,
    pcg_iterations, trials=[per trial: lam, temp, scale, rho, accepted, pcg_*, step bounds], iters=[trials per iteration],
    states=[(poses, points, chi2) after each iteration])."""
    P = P.with_state(P.poses, P.points)
    chi2 = P.chi2()
    out = dict(chi2_before=chi2, trials=[], iters=[], pcg_iterations=0)
    lam, ni, done = 0.0, 2.0, 0
    for i in range(iterations):
        L = P.linearize()
        if i == 0:
            lam = 1e-5 * P.max_diag(L)
        rho, qmax, its = 0.0, 0, []
        while True:
            t = trial(P, L, lam)
            temp = t["temp"]
            rho = (chi2 - temp) / (t["scale"] + 1e-3)
            t["chi2"], t["rho"] = chi2, rho
            t["bound_c"], t["bound_p"] = step_bound(t)
            t["certified"] = (abs(rho) > RHO_BAND and abs(chi2 - temp) > CHI2_BAND * abs(chi2)) or not t["ok"]
            out["pcg_iterations"] += t["pcg_iterations"]
            if rho > 0 and math.isfinite(temp):
                alpha = 1.0 - math.pow(2 * rho - 1, 3)
                alpha = min(alpha, 2.0 / 3.0)
                lam *= max(1.0 / 3.0, alpha)
                ni = 2.0
                chi2 = temp
                P = P.with_state(t["poses"], t["points"])
                t["accepted"] = True
            else:
                lam *= ni
                ni *= 2
                t["accepted"] = False
            for k in ("poses", "points"):
                t.pop(k)
            its.append(t)
            out["trials"].append(t)
            qmax += 1
            if not math.isfinite(lam):
                break
            if not (rho < 0 and qmax < 10):
                break
        out["iters"].append(its)
        out.setdefault("states", []).append((P.poses, P.points, chi2))
        done += 1
        if qmax == 10 or rho == 0:
            break
    out.update(poses=P.poses, points=P.points, chi2=chi2, lm_iterations=done)
    return out


def all_certified(res):
    return all(t["certified"] and t["pcg_certified"] for t in res["trials"])


def certified_prefix(res):
    """how many leading LM iterations have every trial's decision and PCG stop certified"""
    k = 0
    for its in res["iters"]:
        if not all(t["certified"] and t["pcg_certified"] for t in its):
            break
        k += 1
    return k


def iteration_bound(its):
    """(camera, point) step bound of one LM iteration: the accepted trial's, 0 when every trial was rejected"""
    acc = [t for t in its if t["accepted"]]
    return (acc[0]["bound_c"], acc[0]["bound_p"]) if acc else (0.0, 0.0)


# ---- problems -----------------------------------------------------------------------------------------------------
def _quat_yaw_pitch(yaw, pitch):
    """rotation about y by yaw, then about x by pitch, as (x, y, z, w)"""
    qy = np.array([0.0, math.sin(yaw / 2), 0.0, math.cos(yaw / 2)])
    qx = np.array([math.sin(pitch / 2), 0.0, 0.0, math.cos(pitch / 2)])
    x1, y1, z1, w1 = qy
    x2, y2, z2, w2 = qx
    return np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                     w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])


def _pose_inv(p):
    R = rot(p[3:])
    return np.concatenate([-R.T @ p[:3], [-p[3], -p[4], -p[5], p[6]]])


def _pose_mul(a, b):
    Ra = rot(a[3:])
    x1, y1, z1, w1 = a[3:]
    x2, y2, z2, w2 = b[3:]
    q = np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                  w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])
    return np.concatenate([a[:3] + Ra @ b[:3], q / np.linalg.norm(q)])


def make_ba_corridor(n_cams=40, n_points=600, window=40, seed=0, *, obs_counts=None, loops=0, hub=None, hub_edges=0,
                     fixed=(0,), no_obs=(), isolated=None, outliers=(), once=0, fixed_only_points=0, duplicates=0,
                     unobserved=0, edges=True, pose_noise=0.02, rot_noise_deg=1.0, point_noise=0.02, pix_noise=0.5,
                     depth_sigma=0.003, edge_noise=0.005, shallow=0, K4=(525.0, 525.0, 319.5, 239.5)):
    """Cameras along a corridor (x axis) looking at a wall of landmarks (z in [2.5, 4.5]); camera c observes the `window`
    landmarks nearest to it along x, so every landmark is seen by a few neighbouring cameras and the reduced camera system is
    banded and well conditioned at hundreds of cameras.
      obs_counts   {camera: count}: that camera observes exactly `count` landmarks (its nearest ones)
      loops        loop-closure edges between cameras 3..12 apart (modulo n_cams), each direction at random (cameras in both
                   edge roles)
      hub, hub_edges   one camera with `hub_edges` extra edges to cameras along the corridor, as i and as j
      fixed        fixed cameras (any positions, e.g. the first, one mid-sequence and the last)
      no_obs       cameras that keep their edges but observe nothing
      isolated     one camera with neither observations nor edges
      outliers     pose-edge indices whose measurement is off by 0.3 m / 0.1 rad (e'We far above the Huber delta)
      once         extra landmarks seen by exactly one (free) camera
      fixed_only_points  extra landmarks seen only by fixed cameras
      duplicates   observations repeated for the same (camera, landmark) with fresh noise
      unobserved   extra landmarks without observations (appended last)
      shallow      landmarks initialised 0.3 m in front of their first observer, up to 0.5 m off its axis (a strongly
                   nonlinear start: the first LM trials at lambda_0 can overshoot)
    Returns the dict layout of synth.make_ba_problem (gt_poses, gt_points, poses, points, fixed, obs_*, K4, ij, meas, info)."""
    from rgbdslam_v2_b200 import synth
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = K4
    spacing = 0.1
    gt = np.zeros((n_cams, 7))
    for c in range(n_cams):
        gt[c, :3] = [spacing * c, 0.05 * math.sin(0.3 * c), 0.03 * math.cos(0.2 * c)]
        gt[c, 3:] = _quat_yaw_pitch(0.05 * math.sin(0.1 * c), 0.03 * math.cos(0.15 * c))
    span = spacing * (n_cams - 1)
    base = n_points
    pts = np.stack([rng.uniform(-0.6, span + 0.6, base), rng.uniform(-0.8, 0.8, base), rng.uniform(2.5, 4.5, base)], 1)
    cam_x = gt[:, 0]
    order = np.argsort(pts[:, 0], kind="stable")
    sel = {}
    no_obs = set(int(c) for c in no_obs)
    for c in range(n_cams):
        if c in no_obs or c == isolated:
            sel[c] = np.zeros(0, np.int64)
            continue
        k = window if obs_counts is None or c not in obs_counts else obs_counts[c]
        dist = np.abs(pts[:, 0] - cam_x[c])
        sel[c] = np.sort(np.argsort(dist, kind="stable")[:k])
    fixed = sorted(set(int(c) for c in fixed))
    free_obs = [c for c in range(n_cams) if c not in fixed and len(sel[c])]
    extra = []                                 # (point, [cameras])
    for _ in range(once):
        c = free_obs[int(rng.integers(len(free_obs)))]
        extra.append((np.array([cam_x[c] + rng.uniform(-0.2, 0.2), rng.uniform(-0.5, 0.5), rng.uniform(2.5, 4.5)]), [c]))
    fobs = [c for c in fixed if len(sel[c])]
    for _ in range(fixed_only_points if fobs else 0):
        c = fobs[int(rng.integers(len(fobs)))]
        extra.append((np.array([cam_x[c] + rng.uniform(-0.2, 0.2), rng.uniform(-0.5, 0.5), rng.uniform(2.5, 4.5)]), [c]))
    oc, op = [], []
    for c in range(n_cams):
        oc.extend([c] * len(sel[c])); op.extend(sel[c].tolist())
    for k, (p, cams) in enumerate(extra):
        for c in cams:
            oc.append(c); op.append(base + k)
    if extra:
        pts = np.vstack([pts, np.array([p for p, _ in extra])])
    oc, op = np.array(oc, np.int64), np.array(op, np.int64)
    if duplicates and len(oc):
        dup = rng.choice(len(oc), duplicates, replace=False)
        oc, op = np.concatenate([oc, oc[dup]]), np.concatenate([op, op[dup]])
    perm = rng.permutation(len(oc))        # observations interleaved across cameras and points
    oc, op = oc[perm], op[perm]
    n_seen = len(pts)
    if unobserved:
        pts = np.vstack([pts, np.stack([rng.uniform(0, span + 0.1, unobserved), rng.uniform(-0.5, 0.5, unobserved),
                                        rng.uniform(2.5, 4.5, unobserved)], 1)])
    uvd = np.zeros((len(oc), 3))
    if len(oc):
        R = rot(gt[oc, 3:])
        pc = np.einsum("nji,nj->ni", R, pts[op] - gt[oc, :3])
        uvd[:, 0] = fx * pc[:, 0] / pc[:, 2] + cx + rng.normal(0, pix_noise, len(oc))
        uvd[:, 1] = fy * pc[:, 1] / pc[:, 2] + cy + rng.normal(0, pix_noise, len(oc))
        uvd[:, 2] = pc[:, 2] + rng.normal(0, depth_sigma, len(oc))
    init = gt.copy()
    for c in range(n_cams):
        if c in fixed:
            continue
        d = np.concatenate([rng.normal(0, pose_noise, 3), np.deg2rad(rot_noise_deg) / 2 * rng.normal(0, 1, 3)])
        init[c] = _pose_mul(gt[c], np.concatenate([d[:3], d[3:], [math.sqrt(max(0.0, 1 - d[3:] @ d[3:]))]]))
    p0 = pts.copy()
    p0[:n_seen] += rng.normal(0, point_noise, (n_seen, 3))
    if shallow and len(op):
        for p in rng.choice(np.unique(op), shallow, replace=False):
            c = oc[np.nonzero(op == p)[0][0]]
            off = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), 0.3])
            p0[p] = init[c, :3] + rot(init[c, 3:]) @ off
    fx_ = np.zeros(n_cams, np.uint8); fx_[fixed] = 1
    out = dict(gt_poses=gt, gt_points=pts, poses=init, points=p0, fixed=fx_, obs_cam=oc.astype(np.int32), obs_point=op.astype(np.int32),
               obs_uvd=uvd, obs_info3=synth.landmark_information(uvd[:, 2], sigma_depth=depth_sigma / 4.0) if len(oc) else
               np.zeros((0, 3)), K4=np.array(K4, np.float64))
    if edges:
        pairs = [(c, c + 1) for c in range(n_cams - 1) if isolated not in (c, c + 1)]
        if isolated is not None and 0 < isolated < n_cams - 1:
            pairs.append((isolated - 1, isolated + 1))
        cand = [c for c in range(n_cams) if c != isolated]
        for _ in range(loops):
            a = cand[int(rng.integers(len(cand)))]
            b = (a + int(rng.integers(3, 13))) % n_cams
            if abs(a - b) < 2 or b == isolated:
                continue
            pairs.append((a, b) if rng.random() < 0.5 else (b, a))
        if hub is not None:
            others = [c for c in cand if c != hub]
            for k, c in enumerate(rng.choice(others, min(hub_edges, len(others)), replace=False)):
                pairs.append((hub, int(c)) if k % 2 == 0 else (int(c), hub))
        ij, meas, info = [], [], []
        outliers = set(int(k) for k in outliers)
        for k, (i, j) in enumerate(pairs):
            rel = _pose_mul(_pose_inv(gt[i]), gt[j])
            s = (0.3, 0.05) if k in outliers else (edge_noise, edge_noise / 2)
            d = np.concatenate([rng.normal(0, s[0], 3), rng.normal(0, s[1], 3)])
            rel = _pose_mul(rel, np.concatenate([d, [math.sqrt(1 - d[3:] @ d[3:])]]))
            ij.append([i, j]); meas.append(rel); info.append((np.eye(6) * 400.0).reshape(-1))
        out.update(ij=np.array(ij, np.int32).reshape(-1, 2), meas=np.array(meas).reshape(-1, 7),
                   info=np.array(info).reshape(-1, 36))
    return out


# The shapes and topologies the GPU tests run (tests/test_ba_exact_cpu.py asserts what each one reaches).  Kernel boundaries:
# 128 points per CTA (ba_points / ba_pt_gather / ba_pt_update), 8 cameras per CTA (ba_cams / ba_cam_apply), a warp per camera
# striding its observations and pose-edge incidences by 32, one 1024-thread CTA over 6 n_cams unknowns (ba_cg_step: a second
# strided pass from 171 cameras), 256 observations / pose edges per chi2 block.
CASES = {
    "c8_p127": dict(n_cams=8, n_points=127, window=40, obs_counts={2: 31, 3: 32, 4: 33}, seed=1),
    "c9_p128_loops": dict(n_cams=9, n_points=128, window=45, loops=4, seed=2),
    "c17_p129_topology": dict(n_cams=17, n_points=120, window=30, loops=8, hub=8, hub_edges=16, fixed=(0, 9, 16), no_obs=(5,),
                              isolated=12, outliers=(3, 17), once=3, fixed_only_points=2, duplicates=6, unobserved=4, seed=3),
    "c17_p257": dict(n_cams=17, n_points=257, window=60, obs_counts={6: 31, 7: 32, 8: 33}, seed=4),
    "c171_topology": dict(n_cams=171, n_points=2000, window=40, obs_counts={85: 1100}, loops=60, hub=100, hub_edges=40,
                          fixed=(0, 90, 170), no_obs=(20, 21), isolated=60, outliers=(5, 180), once=10, fixed_only_points=5,
                          duplicates=30, unobserved=6, seed=5),
    "c200": dict(n_cams=200, n_points=3000, window=40, obs_counts={120: 1050}, loops=60, hub=50, hub_edges=36,
                 fixed=(0, 100, 199), seed=6),
    "pose_edges_only": dict(n_cams=20, n_points=0, window=0, loops=6, unobserved=5, seed=7),
    "no_pose_edges": dict(n_cams=9, n_points=150, window=50, edges=False, seed=8),
    "first_trial_rejected": dict(n_cams=12, n_points=200, window=50, loops=3, shallow=5, seed=0),
}


def coverage(d):
    """the counts a generator configuration is meant to reach"""
    nc, npt = len(d["poses"]), len(d["points"])
    oc, op = np.asarray(d["obs_cam"]), np.asarray(d["obs_point"])
    per_cam = np.bincount(oc, minlength=nc)
    per_pt = np.bincount(op, minlength=npt)
    ij = np.asarray(d.get("ij", np.zeros((0, 2), np.int32))).reshape(-1, 2)
    inc = np.bincount(ij.reshape(-1), minlength=nc) if len(ij) else np.zeros(nc, np.int64)
    fixed = np.asarray(d["fixed"]).astype(bool)
    pairs = oc.astype(np.int64) * max(npt, 1) + op
    return dict(n_cams=nc, n_points=npt, n_obs=len(oc), n_edges=len(ij), per_cam=per_cam, per_pt=per_pt, incidences=inc,
                max_incidences=int(inc.max(initial=0)), duplicates=len(pairs) - len(np.unique(pairs)),
                seen_once=int((per_pt == 1).sum()), unobserved=int((per_pt == 0).sum()),
                fixed_only=int(sum(1 for p in range(npt) if per_pt[p] and fixed[oc[op == p]].all())),
                both_roles=int(sum(1 for c in range(nc) if (ij[:, 0] == c).any() and (ij[:, 1] == c).any() and
                                   not set(ij[ij[:, 0] == c, 1]) <= {c + 1})),
                loop_edges=int((np.abs(ij[:, 0] - ij[:, 1]) > 1).sum()) if len(ij) else 0,
                fixed_in_edges=int(fixed[ij.reshape(-1)].sum()) if len(ij) else 0,
                isolated=[c for c in range(nc) if per_cam[c] == 0 and inc[c] == 0],
                edges_only=[c for c in range(nc) if per_cam[c] == 0 and inc[c] > 0])
