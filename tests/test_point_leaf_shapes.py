"""The BAL point leaves at every separator width and run shape, held to a componentwise backward-error bound.

The generated BAL graphs (gtsam_b200.datasets.bal) give every point the same number of observations, so a build never mixes
separator widths and a GPU fixture only ever reaches a few instantiations of leaf_point_fused_mma_kernel<DC, NTT, JT>.
`mixed_bal` builds one problem that holds, next to each other:
  * fast-path points (one Point3 frontal, m <= 8 projection factors on distinct cameras) at every m from m_min to m_max,
    on camera sets whose point counts give runs of 1 to 65 points (a run splits at B200_LEAF_RUN_MAX; runs shorter than
    4 mini-batches leave warps idle, 13+ points give a warp a second mini-batch, npts mod 4 covers 0..3);
  * points the generic leaf kernel takes: 9, 12 and 20 observations, two factors on one camera, PriorFactor<Point3> on a
    few observed points, and a point with only a prior (a root clique: nothing to extend-add into).
m_max picks the instantiation: nt8 = ceil((DC m_max + 1) / 8) 8-column strips.  BUILDS reaches all seven.

`check` reads what a solve left behind (the Jacobians, the Hessian diagonal, every clique's conditional [R S d], delta) and
checks in extended precision (np.longdouble), entry by entry, that the conditionals are an exact factorisation of a
slightly perturbed system, with the perturbation bounded by the rounding of the sums that produce each entry:
    point p:   |R_p^T R_p - (H_pp + D_p)|,  |R_p^T S'_p - H_pc|,  |R_p^T d'_p - g_p|
    cameras:   |sum_p S'_p^T S'_p + R_c^T R_c - (H_cc + D_c)|,  |sum_p S'_p^T d'_p + R_c^T d_c - g_c|
each at most tau * M, with M the sum of the absolute values of every term on both sides and tau = 2 K u (u = 2^-53, K the
longest sum that reaches one entry: residual rows + 3 per point at the busiest camera, plus the camera block's Cholesky).
The camera sum runs over every point, so a point's Schur complement that is dropped, doubled or put in the wrong place
fails it.  The back-substitution is held to |R x - d| <= tau_b (|R| |x| + |d|), tau_b = 2 (w_max + 1) u, row by row.
None of these depend on the conditioning of the system.  H and g = A^T b are built from the Jacobians the solve used, so
linearisation is out of the loop.

test_checker_on_oracle proves the checker on the CPU oracle: it passes there, and four small corruptions of the oracle's
factorisation each make it fail.  test_point_leaf_shapes_on_gpu runs every build on the device (own process)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from gtsam_b200 import datasets, problem as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53
LD = np.longdouble

# points per camera set, for every m: runs of 1-3 points (fewer mini-batches than warps), 4-8, 13 and 16 (a warp takes a
# second mini-batch, the mb + 8 prefetch fires), 17, 33, 64 and 65 (65 = 64 + 1 at B200_LEAF_RUN_MAX = 64)
COUNTS = (1, 2, 3, 4, 5, 7, 8, 13, 16, 17, 33, 64, 65)
SMALL_COUNTS = (1, 2, 3, 4, 5, 13, 17)           # the emulated builds (tests/emu/run_scenarios.py)
DC = {"cal3_s2": 6, "bundler": 9}
INSTANTIATIONS = {6: (4, 5, 7), 9: (4, 5, 7, 10)}  # NTT of leaf_point_fused_mma_kernel<DC, NTT, JT> (engine.cu)
# (camera model, m_max): every instantiation once
BUILDS = [("cal3_s2", 5), ("cal3_s2", 6), ("cal3_s2", 7), ("cal3_s2", 8), ("bundler", 3), ("bundler", 4), ("bundler", 6),
          ("bundler", 8)]
# undamped solves need every point observed twice (a point seen by one camera is rank 2)
UNDAMPED_BUILDS = [("cal3_s2", 6), ("bundler", 4)]


def instantiation(model, m_max):
    """<DC, NTT> the fused point-leaf kernel is launched with for a build whose widest fast-path point has m_max cameras."""
    dc = DC[model]
    nt8 = (dc * m_max + 1 + 7) // 8
    return dc, next(t for t in INSTANTIATIONS[dc] if nt8 <= t)


def mixed_bal(model, m_max, m_min=1, counts=COUNTS, off_path=True, ncams=28, seed=3):
    """A BAL problem whose points have explicit camera sets (see the module docstring).  Geometry as datasets.bal: cameras
    on a radius-20 circle looking at the origin, points in +-3, so every point is in front of every camera; priors on
    cameras 0 and 1; Schur ordering (points, then cameras)."""
    rng = np.random.default_rng(seed)
    sets, used = [], set()

    def pick(m):
        # a new camera set with a camera outside the last four: a point seen only by cameras of the root clique would be
        # merged into it (its separator would be all of the root's variables) instead of being a leaf
        while True:
            cs = tuple(sorted(rng.choice(ncams, size=m, replace=False).tolist()))
            if cs not in used and cs[0] < ncams - 4:
                used.add(cs)
                return list(cs)
    for m in range(m_min, m_max + 1):
        for n in counts:
            sets += [pick(m)] * n
    prior_pts = []
    if off_path:
        for m in (9, 12, 20):                                  # more observations than the fast path takes
            sets.append(pick(m))
        a, b, c = pick(3)
        sets.append([a, b, c, a])                              # two factors on one camera
        for m in (1, 3, max(m_min, 2)):                        # observed points with a PriorFactor<Point3>
            prior_pts.append(len(sets))
            sets.append(pick(m))
        prior_pts.append(len(sets))
        sets.append([])                                        # a prior only: a root leaf clique
    npts = len(sets)
    th = 2 * np.pi * np.arange(ncams) / ncams
    eye = np.stack([20 * np.cos(th), 20 * np.sin(th), 2 * np.sin(3 * th)], -1)
    Rc, tc = datasets.lookat_pose(eye, np.zeros(3), np.array([0.0, 0, 1.0]))
    pts = rng.uniform(-3, 3, size=(npts, 3))
    pid = np.array([p for p, cs in enumerate(sets) for _ in cs], dtype=np.int64)
    cid = np.array([c for cs in sets for c in cs], dtype=np.int64)
    q = np.einsum("nji,nj->ni", Rc[cid], pts[pid] - tc[cid])
    assert np.all(q[:, 2] > 0)
    pn = q[:, :2] / q[:, 2:3]
    noise = rng.normal(size=pn.shape)
    Rp, tp = datasets.se3_exp(rng.normal(size=(ncams, 6)) * 0.01)
    R0, t0 = datasets.pose_compose(Rc, tc, Rp, tp)
    pts0 = pts + rng.normal(size=pts.shape) * 0.05
    keys = np.stack([cid, ncams + pid], -1)
    order = np.concatenate([ncams + np.arange(npts), np.arange(ncams)])
    if model == "cal3_s2":
        K = np.array([[500.0, 500.0, 0.0, 320.0, 240.0]])
        z = np.stack([500 * pn[:, 0] + 320, 500 * pn[:, 1] + 240], -1) + noise
        cams = datasets.pack_pose(R0, t0)
        cam_type = P.VAR_POSE3
        proj = P.FactorGroup(P.FACTOR_PROJECTION_CAL3S2, keys, z, P.NOISE_ISOTROPIC, np.array([1.0]))
        prior = P.FactorGroup(P.FACTOR_PRIOR_POSE3, np.array([[0], [1]]), datasets.pack_pose(Rc[:2], tc[:2]),
                              P.NOISE_ISOTROPIC, np.array([0.1]))
        cal = K
    else:
        f, k1, k2 = 500.0, -0.02, 0.002
        r2 = np.sum(pn * pn, -1, keepdims=True)
        z = f * (1 + (k1 + k2 * r2) * r2) * pn + noise
        intr = np.tile(np.array([f, k1, k2, 0.0, 0.0]), (ncams, 1))
        cams = np.concatenate([datasets.pack_pose(R0, t0), intr], -1)
        gtc = np.concatenate([datasets.pack_pose(Rc, tc), intr], -1)
        cam_type = P.VAR_CAM_BUNDLER
        proj = P.FactorGroup(P.FACTOR_SFM_BUNDLER, keys, z, P.NOISE_ISOTROPIC, np.array([1.0]))
        prior = P.FactorGroup(P.FACTOR_PRIOR_CAM_BUNDLER, np.array([[0], [1]]), gtc[:2], P.NOISE_ISOTROPIC, np.array([0.1]))
        cal = np.zeros((0, 5))
    groups = [proj, prior]
    if prior_pts:
        pp = np.array(prior_pts)
        groups.append(P.FactorGroup(P.FACTOR_PRIOR_POINT3, (ncams + pp)[:, None], pts[pp] + rng.normal(size=(pp.size, 3)) * 0.1,
                                    P.NOISE_DIAGONAL, np.array([0.1, 0.2, 0.3])))
    var_type = np.concatenate([np.full(ncams, cam_type), np.full(npts, P.VAR_POINT3)])
    pr = P.Problem(var_type, np.concatenate([cams.ravel(), pts0.ravel()]), order, groups, cal,
                   name=f"mixed_bal_{model}_m{m_min}-{m_max}")
    pr.meta = dict(model=model, m_min=m_min, m_max=m_max, ncams=ncams, npoints=npts)
    return pr


def tau(prob):
    """(tau, tau_b): K = the most products summed into one entry of the camera block (2 rows per observation + the prior's
    rows at a camera, 3 per point that sees it, then the Cholesky of the camera block) + 1."""
    dims, cam = prob.var_dims, prob.var_type != P.VAR_POINT3
    rows = np.zeros(prob.nvars, dtype=np.int64)
    seen = [set() for _ in range(prob.nvars)]
    for g in prob.groups:
        d = P.FACTOR_DIM[g.type]
        for a in range(g.keys.shape[1]):
            np.add.at(rows, g.keys[:, a], d)
        if g.keys.shape[1] == 2:
            for c, p in g.keys:
                seen[c].add(p)
    ncd = int(dims[cam].sum())
    K = max(int(rows[v]) + 3 * len(seen[v]) for v in np.where(cam)[0]) + ncd + 1
    return 2 * K * U, K


def readout(be, prob):
    """Everything the checks read from a solved problem (DeviceProblem or OracleProblem), each read once."""
    dev = hasattr(be.L, "b200_get_conditional")
    fp, fv, sp, sv, par = be.cliques()
    dims = prob.var_dims
    conds = []
    for c in range(len(par)):
        f, s = int(dims[fv[fp[c]:fp[c + 1]]].sum()), int(dims[sv[sp[c]:sp[c + 1]]].sum())
        buf = np.zeros(f * (f + s + 1))
        ptr = buf.ctypes.data_as(C.POINTER(C.c_double))
        if dev:
            rc = be.L.b200_get_conditional(be.h, c, ptr)
            assert rc == 0, (c, rc)
        else:
            be.L.orc_get_conditional(be.h, c, ptr)
        conds.append(buf.reshape(f + s + 1, f).T)
    return dict(J=[be.get_jacobians(gi) for gi in range(len(prob.groups))], hdiag=be.hessian_diagonal(),
                cliques=(fp, fv, sp, sv, par), conds=conds, delta=be.get_delta())


def point_cliques(prob, rd):
    """Clique ids of the point cliques (one Point3 frontal), in clique order."""
    fp, fv, _, _, par = rd["cliques"]
    return [c for c in range(len(par)) if fp[c + 1] - fp[c] == 1 and prob.var_type[fv[fp[c]]] == P.VAR_POINT3]


def _ratio(res, M, t):
    """max |res| / (t M); an entry whose bound is zero must be exactly zero."""
    res, M = np.abs(res), t * M
    if np.any((M == 0) & (res != 0)):
        return np.inf
    nz = M > 0
    return float((res[nz] / M[nz]).max()) if nz.any() else 0.0


def check(prob, rd, lam, diagonal, min_diag=1e-6, max_diag=1e32, drop=None):
    """Worst |residual| / bound of every check (module docstring); all <= 1 passes.  `drop`: a point clique left out of
    the camera sums (a stand-in for a point missing from its run's Schur complement)."""
    t, _ = tau(prob)
    dims, dof = prob.var_dims, prob.dof_offsets()
    is_pt = prob.var_type == P.VAR_POINT3
    cams = np.where(~is_pt)[0]
    ccol = np.full(prob.nvars, -1, dtype=np.int64)           # first column of a camera in the camera block
    ccol[cams] = np.concatenate([[0], np.cumsum(dims[cams])[:-1]])
    ncd = int(dims[cams].sum())
    fp, fv, sp, sv, par = rd["cliques"]
    pcl = point_cliques(prob, rd)
    npt = len(pcl)
    pvar = np.array([fv[fp[c]] for c in pcl], dtype=np.int64)
    pidx = np.full(prob.nvars, -1, dtype=np.int64)
    pidx[pvar] = np.arange(npt)
    assert npt == int(is_pt.sum())
    # per point: [R S' d'] with S' in the point's own separator columns (padded to the widest), and where they go
    seps = [[int(v) for v in sv[sp[c]:sp[c + 1]]] for c in pcl]
    smax = max(1, max(int(dims[s].sum()) if s else 0 for s in seps))
    R = np.zeros((npt, 3, 3), dtype=LD)
    S = np.zeros((npt, 3, smax), dtype=LD)
    d = np.zeros((npt, 3), dtype=LD)
    cols = np.zeros((npt, smax), dtype=np.int64)              # camera-block column of every separator column
    slot = {}                                                 # (point index, camera) -> first separator column
    for i, (c, sep) in enumerate(zip(pcl, seps)):
        cd = rd["conds"][c].astype(LD)
        w = cd.shape[1] - 4
        assert all(not is_pt[v] for v in sep), "a point clique's separator holds a point"
        R[i], S[i, :, :w], d[i] = cd[:, :3], cd[:, 3:3 + w], cd[:, -1]
        o = 0
        for v in sep:
            slot[(i, v)] = o
            cols[i, o:o + dims[v]] = ccol[v] + np.arange(dims[v])
            o += dims[v]
    # H = sum_f J_f^T J_f and |H| = sum_f |J_f|^T |J_f|, in the same layout: point blocks, point-camera (separator
    # columns), camera block; g = A^T b
    Hpp, aHpp = np.zeros((npt, 3, 3), dtype=LD), np.zeros((npt, 3, 3), dtype=LD)
    Hpc, aHpc = np.zeros((npt, 3, smax), dtype=LD), np.zeros((npt, 3, smax), dtype=LD)
    Hcc, aHcc = np.zeros((ncd, ncd), dtype=LD), np.zeros((ncd, ncd), dtype=LD)
    gp, agp = np.zeros((npt, 3), dtype=LD), np.zeros((npt, 3), dtype=LD)
    gc, agc = np.zeros(ncd, dtype=LD), np.zeros(ncd, dtype=LD)
    for gi, g in enumerate(prob.groups):
        J = rd["J"][gi].astype(LD)
        b, aJ = J[:, :, -1], np.abs(J)
        vt = P.FACTOR_VAR_TYPES[g.type]
        c0 = np.concatenate([[0], np.cumsum([P.VAR_DIM[x] for x in vt])])
        for a in range(len(vt)):
            Aa, aAa, ka, da = J[:, :, c0[a]:c0[a + 1]], aJ[:, :, c0[a]:c0[a + 1]], g.keys[:, a], P.VAR_DIM[vt[a]]
            ga, aga = np.einsum("fki,fk->fi", Aa, b), np.einsum("fki,fk->fi", aAa, np.abs(b))
            if vt[a] == P.VAR_POINT3:
                np.add.at(gp, pidx[ka], ga); np.add.at(agp, pidx[ka], aga)
            else:
                ix = ccol[ka][:, None] + np.arange(da)
                np.add.at(gc, ix, ga); np.add.at(agc, ix, aga)
            for bb in range(len(vt)):
                Ab, aAb, kb, db = J[:, :, c0[bb]:c0[bb + 1]], aJ[:, :, c0[bb]:c0[bb + 1]], g.keys[:, bb], P.VAR_DIM[vt[bb]]
                B, aB = np.einsum("fki,fkj->fij", Aa, Ab), np.einsum("fki,fkj->fij", aAa, aAb)
                if vt[a] == P.VAR_POINT3 and vt[bb] == P.VAR_POINT3:
                    np.add.at(Hpp, pidx[ka], B); np.add.at(aHpp, pidx[ka], aB)
                elif vt[a] == P.VAR_POINT3:
                    pi = pidx[ka]
                    o = np.array([slot[(int(x), int(v))] for x, v in zip(pi, kb)], dtype=np.int64)
                    ix = (pi[:, None, None], np.arange(3)[None, :, None], (o[:, None] + np.arange(db))[:, None, :])
                    np.add.at(Hpc, ix, B); np.add.at(aHpc, ix, aB)
                elif vt[bb] != P.VAR_POINT3:
                    ix = ((ccol[ka][:, None] + np.arange(da))[:, :, None], (ccol[kb][:, None] + np.arange(db))[:, None, :])
                    np.add.at(Hcc, ix, B); np.add.at(aHcc, ix, aB)
    # damping D: lambda (additive) or lambda * clip(diag H) (diagonal), the device's / oracle's own diagonal of H
    D = np.zeros(int(dof[-1]), dtype=LD)
    if lam > 0:
        D[:] = LD(lam) * (np.clip(rd["hdiag"], min_diag, max_diag).astype(LD) if diagonal else LD(1))
    Dp = D[dof[pvar][:, None] + np.arange(3)]
    Dc = np.concatenate([D[dof[v]:dof[v] + dims[v]] for v in cams])
    out = {}
    aR, aS, ad = np.abs(R), np.abs(S), np.abs(d)
    RtR, aRtR = np.einsum("pki,pkj->pij", R, R), np.einsum("pki,pkj->pij", aR, aR)
    eye3 = np.eye(3, dtype=LD)
    out["R'R=Hpp+D"] = _ratio(RtR - Hpp - Dp[:, :, None] * eye3, aRtR + aHpp + Dp[:, :, None] * eye3, t)
    out["R'S=Hpc"] = _ratio(np.einsum("pki,pkj->pij", R, S) - Hpc, np.einsum("pki,pkj->pij", aR, aS) + aHpc, t)
    out["R'd=gp"] = _ratio(np.einsum("pki,pk->pi", R, d) - gp, np.einsum("pki,pk->pi", aR, ad) + agp, t)
    # camera block: the camera cliques' rows [R_c d_c], then sum_p S'^T [S' d'] grouped by separator
    Rc, dcv = np.zeros((ncd, ncd), dtype=LD), np.zeros(ncd, dtype=LD)
    for c in range(len(par)):
        if fp[c + 1] - fp[c] == 1 and is_pt[fv[fp[c]]]:
            continue
        gcols = np.concatenate([ccol[v] + np.arange(dims[v]) for v in list(fv[fp[c]:fp[c + 1]]) + list(sv[sp[c]:sp[c + 1]])])
        cd = rd["conds"][c].astype(LD)
        f = cd.shape[0]
        Rc[np.ix_(gcols[:f], gcols)] = cd[:, :-1]
        dcv[gcols[:f]] = cd[:, -1]
    SS, aSS = Rc.T @ Rc, np.abs(Rc).T @ np.abs(Rc)
    Sd, aSd = Rc.T @ dcv, np.abs(Rc).T @ np.abs(dcv)
    groups = {}
    for i, sep in enumerate(seps):
        if pcl[i] != drop and sep:
            groups.setdefault(tuple(sep), []).append(i)
    for sep, members in groups.items():
        mi = np.array(members)
        w = int(dims[list(sep)].sum())
        gcol = cols[mi[0], :w]
        Sg, aSg = S[mi, :, :w], aS[mi, :, :w]
        SS[np.ix_(gcol, gcol)] += np.einsum("pki,pkj->ij", Sg, Sg)
        aSS[np.ix_(gcol, gcol)] += np.einsum("pki,pkj->ij", aSg, aSg)
        Sd[gcol] += np.einsum("pki,pk->i", Sg, d[mi])
        aSd[gcol] += np.einsum("pki,pk->i", aSg, ad[mi])
    out["S'S+Rc'Rc=Hcc+D"] = _ratio(SS - Hcc - np.diag(Dc), aSS + aHcc + np.diag(Dc), t)
    out["S'd+Rc'dc=gc"] = _ratio(Sd - gc, aSd + agc, t)
    # back-substitution, row by row
    wmax = max(int(c.shape[1]) for c in rd["conds"])
    tb = 2 * (wmax + 1) * U
    x = rd["delta"].astype(LD)
    xp = x[dof[pvar][:, None] + np.arange(3)]
    xc = np.concatenate([x[dof[v]:dof[v] + dims[v]] for v in cams])
    xs = xc[cols] * (np.arange(smax)[None, :] < np.array([int(dims[s].sum()) if s else 0 for s in seps])[:, None])
    out["back_points"] = _ratio(np.einsum("pij,pj->pi", R, xp) + np.einsum("pij,pj->pi", S, xs) - d,
                                np.einsum("pij,pj->pi", aR, np.abs(xp)) + np.einsum("pij,pj->pi", aS, np.abs(xs)) + ad, tb)
    rows = np.abs(Rc).sum(1) > 0
    out["back_cameras"] = _ratio((Rc @ xc - dcv)[rows], (np.abs(Rc) @ np.abs(xc) + np.abs(dcv))[rows], tb)
    return out


def linear_error(prob, rd):
    """0.5 |A delta - b|^2 in extended precision, from the Jacobians the solve used."""
    dof = prob.dof_offsets()
    x = rd["delta"].astype(LD)
    e = LD(0)
    for gi, g in enumerate(prob.groups):
        J = rd["J"][gi].astype(LD)
        r = -J[:, :, -1]
        c0 = 0
        for a, vt in enumerate(P.FACTOR_VAR_TYPES[g.type]):
            n = P.VAR_DIM[vt]
            r = r + np.einsum("fkj,fj->fk", J[:, :, c0:c0 + n], x[dof[g.keys[:, a]][:, None] + np.arange(n)])
            c0 += n
        e += (r * r).sum()
    return float(e / 2)


def fmt(ratios):
    return "  ".join(f"{k} {v:.3g}" for k, v in ratios.items())


# ---- the checker proven on the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,m_max", [("cal3_s2", 6), ("bundler", 4)])
def test_checker_on_oracle(model, m_max):
    """The checker passes on the CPU oracle's factorisation, and each of four corruptions of it fails the checker."""
    from oracle import oracle_py as O
    prob = mixed_bal(model, m_max, counts=SMALL_COUNTS)
    orc = O.OracleProblem(prob)
    orc.linearize()
    for lam, diag in ((1e-2, False), (1e-3, True)):
        st, e0, e1, _ = orc.solve(lam, diag)
        assert st == 0
        rd = readout(orc, prob)
        ok = check(prob, rd, lam, diag)
        print(model, m_max, lam, diag, fmt(ok))
        assert max(ok.values()) <= 1.0, ok
        assert abs(e1 - linear_error(prob, rd)) <= 1e-9 * e0
    # corruptions of the last (diagonally damped) solve
    pcl = point_cliques(prob, rd)
    fp, fv, sp, sv, _ = rd["cliques"]
    wide = [c for c in pcl if sp[c + 1] - sp[c] >= 2]
    c = wide[len(wide) // 2]

    def fails(rd2, **kw):
        r = check(prob, rd2, lam, diag, **kw)
        return max(r.values()) > 1.0, r

    # 1. one entry of one point's S' off by 1e-8 relative
    bad = dict(rd, conds=list(rd["conds"]))
    cd = bad["conds"][c].copy()
    j = 3 + int(np.argmax(np.abs(cd[:, 3:-1]).max(0)))
    i = int(np.argmax(np.abs(cd[:, j])))
    cd[i, j] *= 1 + 1e-8
    bad["conds"][c] = cd
    f, r = fails(bad)
    assert f and r["R'S=Hpc"] > 1.0, r
    # 2. one point missing from the camera sums
    f, r = fails(rd, drop=c)
    assert f and r["S'S+Rc'Rc=Hcc+D"] > 1.0, r
    # 3. two camera slots of one point's S' swapped
    bad = dict(rd, conds=list(rd["conds"]))
    cd = rd["conds"][c].copy()
    dc = DC[model]
    cd[:, 3:3 + dc], cd[:, 3 + dc:3 + 2 * dc] = rd["conds"][c][:, 3 + dc:3 + 2 * dc], rd["conds"][c][:, 3:3 + dc]
    bad["conds"][c] = cd
    f, r = fails(bad)
    assert f and r["R'S=Hpc"] > 1.0, r
    # 4. one point's x_p off by 1e-8 relative (the point whose row residual is dominated by R_p x_p)
    dof, dims = prob.dof_offsets(), prob.var_dims
    x = rd["delta"]
    best, pv = -1.0, None
    for q in pcl:
        v = int(fv[fp[q]])
        cd = rd["conds"][q]
        xs = np.concatenate([[0.0]] + [x[dof[u]:dof[u] + dims[u]] for u in sv[sp[q]:sp[q + 1]]])[1:]
        xp = x[dof[v]:dof[v] + 3]
        share = np.abs(cd[:, :3] @ xp).max() / (np.abs(cd[:, :3]) @ np.abs(xp) + np.abs(cd[:, 3:-1]) @ np.abs(xs) + np.abs(cd[:, -1])).max()
        if share > best:
            best, pv = share, v
    bad = dict(rd, delta=rd["delta"].copy())
    bad["delta"][dof[pv]:dof[pv] + 3] *= 1 + 1e-8
    f, r = fails(bad)
    assert f and r["back_points"] > 1.0, r


def test_builds_reach_every_instantiation():
    """The builds below launch every <DC, NTT> of the fused point-leaf kernel; the generator's shapes are what they claim."""
    got = {instantiation(m, k) for m, k in BUILDS}
    assert got == {(dc, t) for dc, ts in INSTANTIATIONS.items() for t in ts}, got
    prob = mixed_bal("bundler", 8)
    g = prob.groups[0]
    obs = np.bincount(g.keys[:, 1] - prob.meta["ncams"], minlength=prob.meta["npoints"])
    fast = [p for p in range(prob.meta["npoints"]) if 1 <= obs[p] <= 8 and len(set(g.keys[g.keys[:, 1] == prob.meta["ncams"] + p, 0])) == obs[p]]
    assert set(obs[fast]) == set(range(1, 9))
    assert {9, 12, 20, 0} <= set(obs.tolist())
    assert sorted({n % 4 for n in COUNTS}) == [0, 1, 2, 3]


# ---- the GPU test ----------------------------------------------------------------------------------------------------------
SCRIPT = r"""
import os, sys, time
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import util
import test_point_leaf_shapes as T
from gtsam_b200 import capi
from oracle import oracle_py as O
ctx = capi.Context(0)
print("instantiations launched:")
for model, m_max in T.BUILDS:
    print("  %-8s m_max %d  -> leaf_point_fused_mma_kernel<%d, %d>" % ((model, m_max) + T.instantiation(model, m_max)))
worst, cells, t0 = {{}}, 0, time.time()
plan = [(b, False) for b in T.BUILDS] + [(b, True) for b in T.UNDAMPED_BUILDS]
for (model, m_max), undamped in plan:
    prob = T.mixed_bal(model, m_max, m_min=2 if undamped else 1)
    solves = ((0.0, False),) if undamped else ((1e-2, False), (1e-3, True))
    for f32 in (False, True):
        ref = {{}}
        if not undamped:
            orc = O.OracleProblem(prob)
            orc.set_jacobian_precision(f32)
            orc.linearize()
            for lam, diag in solves:
                assert orc.solve(lam, diag)[0] == 0
                ref[(lam, diag)] = orc.get_delta()
            del orc
        for run in (None, 64):
            if run:
                os.environ["B200_LEAF_RUN_MAX"] = str(run)
            try:
                dev = capi.DeviceProblem(ctx, prob)
                split = capi.DeviceProblem(ctx, prob) if not undamped else None
            finally:
                os.environ.pop("B200_LEAF_RUN_MAX", None)
            if split:
                split.set_tuning("schur_mma", 0)
            for d in (dev, split):
                if d:
                    d.set_jacobian_precision(f32); d.linearize()
            for lam, diag in solves:
                st, e0, e1, _ = dev.solve(lam, diag)
                assert st == 0, (model, m_max, f32, run, lam, diag, st)
                rd = T.readout(dev, prob)
                r = T.check(prob, rd, lam, diag)
                le = abs(e1 - T.linear_error(prob, rd)) / (1e-9 * e0)
                cell = "%s m%d-%d %s run %s lam %g %s" % (model, 2 if undamped else 1, m_max, "fp32" if f32 else "fp64", run or "default", lam, "diag" if diag else "add")
                print(cell, " ", T.fmt(r), " e1 %.3g" % le, flush=True)
                for k, v in list(r.items()) + [("e1", le)]:
                    worst[k] = max(worst.get(k, 0.0), v)
                assert max(r.values()) <= 1.0 and le <= 1.0, (cell, r, le)
                if lam > 0:
                    tol = 1e-5 if f32 else 1e-8
                    rel = util.rel2(rd["delta"], ref[(lam, diag)])
                    assert rel <= tol, (cell, "delta vs oracle", rel)
                if split and not diag:
                    assert split.solve(lam, diag)[0] == 0
                    pc = T.point_cliques(prob, rd)
                    other = T.readout(split, prob)
                    bad = [c for c in pc if not np.array_equal(rd["conds"][c], other["conds"][c])]
                    assert not bad, (cell, "point conditionals differ from the split path", len(bad), len(pc))
                cells += 1
            dev.close()
            if split:
                split.close()
print("worst residual / bound over %d cells (%.0f s):" % (cells, time.time() - t0))
for k, v in worst.items():
    print("  %-18s %.3g" % (k, v))
print("SHAPES_OK", cells)
"""


@pytest.mark.gpu
def test_point_leaf_shapes_on_gpu():
    """Every build of BUILDS (and UNDAMPED_BUILDS at lambda = 0) on the device: FP64 and FP32 Jacobian storage, the default
    run length and runs of up to 64 points, additive (1e-2) and diagonal (1e-3) damping; every check of `check`, the
    linear error, delta against the oracle (1e-8; FP32 storage: 1e-5 with the oracle in FP32 mode), and the point
    conditionals of the additively damped solve bitwise equal to the split path's (schur_mma = 0).  Own process."""
    try:
        out = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT)], capture_output=True, text=True, timeout=900)
    except subprocess.TimeoutExpired:
        pytest.fail("point-leaf shapes: timed out")
    print(out.stdout)
    lines = [l for l in out.stdout.splitlines() if l.startswith("SHAPES_OK")]
    if not lines:
        pytest.fail("point-leaf shapes: did not complete: " + out.stdout[-2000:] + out.stderr[-3000:])
    assert int(lines[-1].split()[1]) > 0
