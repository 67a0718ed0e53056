"""The dense fronts (front_df_kernel, elim_small_kernel) and their back-substitution (backsub_large_kernel, backsub_small_kernel)
at every tile and block boundary, held to a componentwise backward-error bound over the whole tree.

`front_tree` builds a GaussianFactorGraph whose fronts have chosen shapes: a front of f pivots is a node of variables summing
to f, joined by one dense JacobianFactor (more rows than columns) to a chosen set of variables of a later node (its separator,
of width s).  A node without a separator is a root; its variables also get priors.  What the device eliminates is decided by
the junction tree and by relaxed amalgamation, not by the generator: a front whose separator is the whole of its parent's
clique is merged into it, and amalgamation (on by default, off with B200_NO_AMALGAMATE) merges small and thin fronts.  So
every shape claim below is checked on the supernodes of the host-only symbolic phase (capi.linear_symbolic).  BUILDS reach:
  * f in F_GRID: K = 1..6 pivot blocks of 32, the diagonal block in the first and the second 4-block row tile, a short last
    pivot block of 1 and of 31 rows, and 64-row back-substitution blocks of 1, 31, 32, 33, 63 and 64 rows;
  * s + 1 in S1_GRID (1: a root);
  * nn = f + s + 1 of 47 and 48 below the first dataflow level (elim_small_kernel) and above it (front_df_kernel, then
    backsub_small_kernel), and 49 (the smallest dataflow-only front);
  * thin dataflow fronts (f <= 8, nn > 48), a chain of three dataflow fronts (Schur complements pass from tiles to tiles
    inside one launch), fronts of different shapes on one level, small leaves under dataflow fronts, a forest of two roots,
    and one front given as a HessianFactor.
"graded" is build "level0" with every column of the graph scaled by 10^u, u uniform in [-4, 4] (but the last two pivots of
every front), so that some 32 x 32 diagonal blocks R_bb have condition numbers above 1e8 (3e8 at lambda = 0).

`check` reads what a solve left behind (the whitened Jacobians, every clique's conditional [R S d], delta) and checks in
extended precision (np.longdouble, 64-bit mantissa), entry by entry:
    |U'U - H - D| <= tau (|U|'|U| + |H| + D)          |U'd - g| <= tau (|U|'|d| + |g|)
U and d are the conditionals of every clique, H = sum of A'A over the JacobianFactors + G of the HessianFactors, g = A'b + g,
D the damping (lambda, or lambda clip(diag H)).  tau = 2 K u, u = 2^-53.  An entry of H + D is the sum of one product per
factor row that touches its column, one term per HessianFactor, one Schur-complement term per child front (the extend-add)
and the damping; its partial Cholesky then subtracts one product per earlier pivot, at most the nonzeros of U's column.
So K = max over columns of (nonzeros of U's column + factor rows touching it) + the most children of a supernode + 1.
U'U and |U|'|U| are summed clique by clique (a clique's rows touch only its frontal and separator columns), so a child's
Schur complement that is lost, doubled or extend-added into the wrong slot fails the first check, whatever the conditioning.

Back-substitution, row by row, with tau_b = 2 (w_max + 1) u (w_max the widest conditional):
  * rows solved by substitution (backsub_small_kernel, and the leaf kernels of typed problems):
        |d - U x| <= tau_b (|U| |x| + |d|)
  * rows of the supernodes that go to backsub_large_kernel (`backsub_large`) are solved by multiplying with W ~ R_bb^-1,
    the inverse front_df_kernel leaves behind for every 32-row block b of the front.  A solve by explicit inverse has the
    residual (R_bb W - I) rhs + R_bb (rounding of W rhs), so their bound is the one above plus
        gamma |R_bb| |R_bb^-1| (|d_b| + sum_{j > b} |R_bj| |x_j|),     gamma = 2 * 33 u
    with R_bb^-1 computed in extended precision from the device's own R_bb.  The strict substitution bound of these rows is
    reported as well (the cost of the explicit inverse), but not asserted on.
The device's linear error e1 must match 0.5 |A delta - b|^2 + 0.5 (f - 2 delta'g + delta'G delta) to 1e-9 e0.

test_checker_on_oracle proves the checker on the CPU oracle: it passes there, and four small corruptions each fail the check
they aim at.  test_builds_reach_the_grid checks the shapes on the symbolic phase alone.  test_front_shapes_on_gpu runs every
build on the device (own process), and the "frontshapes" scenario of tests/emu/run_scenarios.py runs a reduced build through
the emulated library."""
import os
import subprocess
import sys

import numpy as np
import pytest

from gtsam_b200 import linear as LN, problem as P
from test_point_leaf_shapes import LD, U, _ratio, readout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_MAX_N = 48          # kSmallMaxN (kernels.cuh): fronts up to this size are one warp per clique
THIN_F = 8                # plan_levels (engine.cu): dataflow fronts of at most 8 pivots are back-substituted one warp each
BLOCK = 32                # kDfB (front_df.cuh): the pivot blocks, and the diagonal blocks W = R_bb^-1 is kept for
LEAF_MAX_F = 6            # kLeafMaxF (kernels.cuh): typed problems' leaves up to this many pivots take the fused leaf kernels
JACOBIAN_MAX_ARITY = 8    # B200_JACOBIAN_MAX_ARITY (include/gtsam_b200.h)
F_GRID = (1, 2, 8, 9, 31, 32, 33, 63, 64, 65, 127, 128, 129, 160, 161)
S1_GRID = (1, 31, 32, 33, 64, 65, 129)
DAMPING = ((0.0, False), (1e-3, False), (1e-2, True))


def _r(node, *ks):
    return [(node, k) for k in ks]


def build_nodes(name):
    """[(node, variable dims, separator)] in elimination order; a separator lists (node, variable index) of later nodes."""
    if name in ("level0", "graded"):
        # one level of fronts of every width under a 161-pivot root (R5 is in no separator: no front is absorbed into
        # the root), and a second root: a forest.  s: R0 = 30, R0+R1 = 31, R2 = 32, R0+R1+R2 = 63, R2+R3 = 64, R0..R4 = 128
        return [("f1", [1], _r("R", 2, 3)), ("f2", [2], _r("R", 0)), ("f8", [8], _r("R", 0, 1, 2)),
                ("f9", [9], _r("R", 0, 1, 2)), ("f31", [31], _r("R", 0, 1)), ("f32", [32], _r("R", 0)),
                ("f33", [33], _r("R", 2)), ("f63", [31, 32], _r("R", 3)), ("f64", [64], _r("R", 2, 3)),
                ("f65", [65], _r("R", 0, 1, 2, 3, 4)), ("n47", [14], _r("R", 2)), ("n48", [15], _r("R", 3)),
                ("n49", [17], _r("R", 0, 1)),
                ("R", [30, 1, 32, 32, 33, 33], []), ("Q", [46], [])]
    if name == "nested":
        # dataflow fronts two and three levels up (M3 -> M1 -> R), every one of them with small leaf children, so that
        # without amalgamation no leaf is wider than 48 and the fronts of nn 47 / 48 sit below the first dataflow level.
        # M2 is a HessianFactor.
        return [("l1", [14], _r("M3", 0)), ("l2", [15], _r("M3", 0)), ("l3", [2], _r("M1", 0)), ("l4", [1], _r("M1", 1)),
                ("l5", [15], _r("M2", 1)), ("l6", [6], _r("M2", 0)),
                ("M3", [32, 128], [("M1", 2), ("R", 0)]), ("M1", [31, 1, 32, 63], _r("R", 0)),
                ("M2", [33, 32, 64], _r("R", 0, 1)), ("R", [32, 32, 64], [])]
    if name == "reduced":
        # f <= 65 (the emulated scenario): the dataflow fronts of "level0" one level up, under a 65-pivot root, each with a
        # small leaf child (so the leaves, nn 47 and 48 among them, go to elim_small_kernel), and a chain m2 -> M -> R
        fronts = [(8, _r("R", 0, 1, 2)), (9, _r("R", 0, 1, 2)), (31, _r("R", 0, 1)), (32, _r("R", 0)), (33, _r("R", 2)),
                  (63, _r("R", 1, 2)), (64, _r("R", 2)), (65, _r("R", 0))]
        leaves = [("l%d" % f, [1 + f % 2], [("f%d" % f, 0)]) for f, _ in fronts]
        return (leaves + [("n47", [14], [("f33", 1)]), ("n48", [15], [("f33", 1)]), ("m2l", [2], [("m2", 0)])] +
                [("f%d" % f, [1, f - 1], sep) for f, sep in fronts] +
                [("m2", [1, 32], [("M", 0), ("R", 0)]), ("M", [31, 1, 32], _r("R", 0)), ("R", [30, 1, 32, 2], [])])
    raise ValueError(name)


BUILDS = ("level0", "nested", "graded")


def front_tree(name, seed=5, nodes=None, graded=None):
    """The LinearProblem of build `name` (module docstring), or of the node list `nodes` (as build_nodes returns) under that
    name; elimination order = node order.  graded: scale the columns as build "graded" does (default: name == "graded")."""
    nodes = build_nodes(name) if nodes is None else nodes
    graded = name == "graded" if graded is None else graded
    rng = np.random.default_rng(seed)
    var, dims = {}, []
    for node, vd, _ in nodes:
        for k, d in enumerate(vd):
            var[(node, k)] = len(dims)
            dims.append(d)
    dof = np.concatenate([[0], np.cumsum(dims)])
    scale = np.ones(dof[-1])
    if graded:
        scale = 10.0 ** rng.uniform(-4, 4, size=dof[-1])
        # the last two pivots of every front stay unscaled: a ratio of 2^12 between them, or a single pivot below 2^-12,
        # is the underconstrained-system test (gtsam's Cholesky), which would report the system as indeterminate
        for node, vd, _ in nodes:
            end = dof[var[(node, len(vd) - 1)] + 1]
            scale[max(0, end - 2):end] = 1.0
    groups, hgroups = [], []

    def jacobian(keys, extra):
        kd = [dims[v] for v in keys]
        cols = np.concatenate([dof[v] + np.arange(dims[v]) for v in keys])
        rows = len(cols) + extra
        A = rng.normal(size=(rows, len(cols))) * scale[cols]
        return kd, np.concatenate([A, rng.normal(size=(rows, 1))], 1)

    for node, vd, sep in nodes:
        keys = [var[(node, k)] for k in range(len(vd))] + [var[r] for r in sep]
        # a node of more than JACOBIAN_MAX_ARITY keys: factors on its first variable and up to 7 more each; eliminating
        # that variable first joins them all into one clique, as one dense factor would
        parts = [keys] if len(keys) <= JACOBIAN_MAX_ARITY else \
            [[keys[0]] + keys[i:i + JACOBIAN_MAX_ARITY - 1] for i in range(1, len(keys), JACOBIAN_MAX_ARITY - 1)]
        for part in parts:
            kd, Ab = jacobian(part, 3)
            if name == "nested" and node == "M2":
                hgroups.append(LN.HessianGroup(kd, np.array([part]), (Ab.T @ Ab)[None]))
            else:
                groups.append(LN.JacobianGroup(Ab.shape[0], kd, np.array([part]), Ab.T[None]))
        if not sep:
            for k in keys:
                kd, Ab = jacobian([k], 2)
                groups.append(LN.JacobianGroup(Ab.shape[0], kd, np.array([[k]]), Ab.T[None]))
    return LN.LinearProblem(np.array(dims), np.arange(len(dims)), groups, hgroups, name="front_tree_" + name)


class env:
    """Environment variables set only around a block (problem creation reads them)."""

    def __init__(self, **kw):
        self.kw = {k: v for k, v in kw.items() if v is not None}

    def __enter__(self):
        os.environ.update(self.kw)

    def __exit__(self, *a):
        for k in self.kw:
            os.environ.pop(k, None)


def supernode_table(sn, dims):
    """Per supernode (f, s, nn, level, first dataflow level of the tree) from (fp, fv, sp, sv, parent)."""
    fp, fv, sp, sv, par = sn[:5]
    nc = len(par)
    f = np.array([int(dims[fv[fp[c]:fp[c + 1]]].sum()) for c in range(nc)])
    s = np.array([int(dims[sv[sp[c]:sp[c + 1]]].sum()) for c in range(nc)])
    lvl = np.zeros(nc, dtype=np.int64)
    for c in range(nc):                 # children have smaller ids than their parents
        if par[c] >= 0:
            lvl[par[c]] = max(lvl[par[c]], lvl[c] + 1)
    nn = f + s + 1
    df_first = int(lvl[nn > SMALL_MAX_N].min()) if (nn > SMALL_MAX_N).any() else 1 << 30
    return dict(f=f, s=s, nn=nn, level=lvl, df_first=df_first, parent=np.asarray(par))


def symbolic(lp, amalgamate=True):
    """The supernodes the device eliminates (host-only symbolic phase)."""
    from gtsam_b200 import capi
    with env(B200_NO_AMALGAMATE=None if amalgamate else "1"):
        return capi.linear_symbolic(lp, with_slots=True)[:5]


def backsub_large(table, no_thin=False, fused_leaf_max_f=0):
    """Supernodes plan_levels (engine.cu) sends to backsub_large_kernel: more than kSmallMaxN = 48 columns and more than
    8 pivots, or any pivot count under B200_NO_THIN_BACKSUB.  (Fronts wider than 48 are always dataflow fronts; typed
    problems' fused leaves, level 0 with at most `fused_leaf_max_f` pivots, take the leaf back-substitution.)"""
    t = table
    fused = (t["level"] == 0) & (t["f"] <= fused_leaf_max_f)
    return set(np.where((t["nn"] > SMALL_MAX_N) & ((t["f"] > THIN_F) | no_thin) & ~fused)[0].tolist())


def _tri_inv(R):
    """Inverse of an upper-triangular longdouble matrix by column substitution (numpy's linalg has no longdouble)."""
    n = R.shape[0]
    X = np.zeros_like(R)
    for i in range(n - 1, -1, -1):
        e = np.zeros(n, dtype=R.dtype)
        e[i] = 1
        X[i] = (e - R[i, i + 1:] @ X[i + 1:]) / R[i, i]
    return X


def _factor_blocks(prob, rd):
    """(J (count, rows, ncols) longdouble, keys, variable dims) of every JacobianFactor group."""
    lin = isinstance(prob, LN.LinearProblem)
    for gi, g in enumerate(prob.groups):
        dims = list(g.dims) if lin else [P.VAR_DIM[t] for t in P.FACTOR_VAR_TYPES[g.type]]
        yield rd["J"][gi].astype(LD), g.keys, dims


def check(prob, rd, lam, diag, sn, large, min_diag=1e-6, max_diag=1e32, drop=None):
    """(worst |residual| / bound of every check, info) (module docstring); all checks <= 1 passes.  sn: the supernodes the
    device eliminated; large: the ones solved by backsub_large_kernel.  info: the strict substitution ratio of those rows and
    the largest condition number (1-norm) of their diagonal blocks.  drop: a clique left out of the clique-by-clique sums."""
    assert np.finfo(LD).nmant >= 63, "np.longdouble is not extended precision here"
    dims, dof = prob.var_dims, prob.dof_offsets()
    n = int(dof[-1])

    def cols_of(vs):
        return np.concatenate([dof[v] + np.arange(dims[v]) for v in vs]).astype(np.int64) if len(vs) else np.zeros(0, np.int64)
    # H, |H|, g = A'b, |g|, and the factor rows touching every column
    H, aH = np.zeros((n, n), dtype=LD), np.zeros((n, n), dtype=LD)
    g, ag = np.zeros(n, dtype=LD), np.zeros(n, dtype=LD)
    rows = np.zeros(n, dtype=np.int64)
    for J, keys, kd in _factor_blocks(prob, rd):
        col = np.concatenate([dof[keys[:, a]][:, None] + np.arange(kd[a]) for a in range(len(kd))], 1)
        A, b = J[:, :, :-1], J[:, :, -1]
        ix = (col[:, :, None], col[:, None, :])
        np.add.at(H, ix, np.einsum("fki,fkj->fij", A, A))
        np.add.at(aH, ix, np.einsum("fki,fkj->fij", np.abs(A), np.abs(A)))
        np.add.at(g, col, np.einsum("fki,fk->fi", A, b))
        np.add.at(ag, col, np.einsum("fki,fk->fi", np.abs(A), np.abs(b)))
        np.add.at(rows, col, J.shape[1])
    for hg in getattr(prob, "hgroups", []):
        for k in range(hg.count):
            col = cols_of(hg.keys[k])
            info = hg.info[k].astype(LD)
            H[np.ix_(col, col)] += info[:-1, :-1]
            aH[np.ix_(col, col)] += np.abs(info[:-1, :-1])
            g[col] += info[:-1, -1]
            ag[col] += np.abs(info[:-1, -1])
            rows[col] += 1
    D = np.zeros(n, dtype=LD)
    if lam > 0:
        D[:] = LD(lam) * (np.clip(rd["hdiag"], min_diag, max_diag).astype(LD) if diag else LD(1))
    # U, d and their clique-by-clique products
    fp, fv, sp, sv, par = rd["cliques"]
    Um, dv = np.zeros((n, n), dtype=LD), np.zeros(n, dtype=LD)
    UtU, aUtU = np.zeros((n, n), dtype=LD), np.zeros((n, n), dtype=LD)
    Utd, aUtd = np.zeros(n, dtype=LD), np.zeros(n, dtype=LD)
    wmax = 0
    for c in range(len(par)):
        fr, cl = cols_of(fv[fp[c]:fp[c + 1]]), cols_of(list(fv[fp[c]:fp[c + 1]]) + list(sv[sp[c]:sp[c + 1]]))
        cd = rd["conds"][c].astype(LD)
        R, d = cd[:, :-1], cd[:, -1]
        wmax = max(wmax, R.shape[1])
        Um[np.ix_(fr, cl)] = R
        dv[fr] = d
        if c == drop:
            continue
        aR = np.abs(R)
        UtU[np.ix_(cl, cl)] += R.T @ R
        aUtU[np.ix_(cl, cl)] += aR.T @ aR
        Utd[cl] += R.T @ d
        aUtd[cl] += aR.T @ np.abs(d)
    kids = np.bincount(np.asarray(sn[4])[np.asarray(sn[4]) >= 0], minlength=len(sn[4]))
    K = int(((Um != 0).sum(0) + rows).max()) + int(kids.max(initial=0)) + 1
    t = 2 * K * U
    out = {}
    out["U'U=H+D"] = _ratio(UtU - H - np.diag(D), aUtU + aH + np.diag(D), t)
    out["U'd=g"] = _ratio(Utd - g, aUtd + ag, t)
    # back-substitution
    tb = 2 * (wmax + 1) * U
    x = rd["delta"].astype(LD)
    res = Um @ x - dv
    M = np.abs(Um) @ np.abs(x) + np.abs(dv)
    extra = np.zeros(n, dtype=LD)
    is_large = np.zeros(n, dtype=bool)
    gamma, kappa = 2 * 33 * U, 0.0
    sfp, sfv = sn[0], sn[1]
    for c in sorted(large):
        idx = cols_of(sfv[sfp[c]:sfp[c + 1]])
        is_large[idx] = True
        for b0 in range(0, len(idx), BLOCK):
            rb = idx[b0:b0 + BLOCK]
            Rbb = Um[np.ix_(rb, rb)]
            aRbb, aWbb = np.abs(Rbb), np.abs(_tri_inv(Rbb))
            off = np.abs(Um[rb])
            off[:, rb] = 0
            extra[rb] = gamma * (aRbb @ (aWbb @ (np.abs(dv[rb]) + off @ np.abs(x))))
            kappa = max(kappa, float(aRbb.sum(0).max() * aWbb.sum(0).max()))
    out["back_subst"] = _ratio(res[~is_large], M[~is_large], tb)
    out["back_large"] = _ratio(res[is_large], tb * M[is_large] + extra[is_large], 1.0) if is_large.any() else 0.0
    info = dict(strict_large=_ratio(res[is_large], M[is_large], tb) if is_large.any() else 0.0, cond_Rbb=kappa)
    return out, info


def linear_error(prob, rd):
    """The graph error at delta in extended precision: 0.5 |A delta - b|^2 per JacobianFactor, 0.5 (f - 2 delta'g +
    delta'G delta) per HessianFactor."""
    dof = prob.dof_offsets()
    x = rd["delta"].astype(LD)
    e = LD(0)
    for J, keys, kd in _factor_blocks(prob, rd):
        col = np.concatenate([dof[keys[:, a]][:, None] + np.arange(kd[a]) for a in range(len(kd))], 1)
        r = np.einsum("fkj,fj->fk", J[:, :, :-1], x[col]) - J[:, :, -1]
        e += (r * r).sum() / 2
    for hg in getattr(prob, "hgroups", []):
        for k in range(hg.count):
            col = np.concatenate([dof[v] + np.arange(prob.var_dims[v]) for v in hg.keys[k]])
            info, xc = hg.info[k].astype(LD), x[col]
            e += (info[-1, -1] - 2 * xc @ info[:-1, -1] + xc @ (info[:-1, :-1] @ xc)) / 2
    return float(e)


def fmt(ratios):
    return "  ".join(f"{k} {v:.3g}" for k, v in ratios.items())


# ---- the checker proven on the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["level0", "nested"])
def test_checker_on_oracle(name):
    """The checker passes on the CPU oracle's factorisation at every damping, and each of four corruptions fails the check
    it aims at."""
    from oracle import oracle_py as O
    lp = front_tree(name)
    sn = symbolic(lp)
    large = backsub_large(supernode_table(sn, lp.var_dims))
    assert large
    orc = O.OracleLinearProblem(lp)
    for lam, diag in DAMPING:
        st, e0, e1, _ = orc.solve(lam, diag)
        assert st == 0
        rd = readout(orc, lp)
        ok, info = check(lp, rd, lam, diag, sn, large)
        print(name, lam, diag, fmt(ok), fmt(info))
        assert max(ok.values()) <= 1.0, ok
        assert abs(e1 - linear_error(lp, rd)) <= 1e-9 * e0
    # corruptions of the last (diagonally damped) solve
    fp, fv, sp, sv, par = rd["cliques"]
    dims, dof = lp.var_dims, lp.dof_offsets()
    nf = [int(dims[fv[fp[c]:fp[c + 1]]].sum()) for c in range(len(par))]
    ns = [int(dims[sv[sp[c]:sp[c + 1]]].sum()) for c in range(len(par))]

    def fails(rd2, key, **kw):
        r, _ = check(lp, rd2, lam, diag, sn, large, **kw)
        return r[key] > 1.0, r

    def with_cond(c, cd):
        bad = dict(rd, conds=list(rd["conds"]))
        bad["conds"][c] = cd
        return bad
    # 1. one entry of a front's R, in the column just after a 32-boundary, off by 1e-8 relative
    c = next(c for c in range(len(par)) if nf[c] > BLOCK)
    cd = rd["conds"][c].copy()
    i = int(np.argmax(np.abs(cd[:BLOCK + 1, BLOCK])))
    cd[i, BLOCK] *= 1 + 1e-8
    f, r = fails(with_cond(c, cd), "U'U=H+D")
    assert f, r
    # 2. one clique left out of the clique-by-clique sums
    f, r = fails(rd, "U'U=H+D", drop=int(np.argmax(ns)))
    assert f, r
    # 3. two separator columns of one conditional swapped
    c = int(np.argmax(ns))
    cd = rd["conds"][c].copy()
    a, b = nf[c], nf[c] + 1
    cd[:, [a, b]] = cd[:, [b, a]]
    f, r = fails(with_cond(c, cd), "U'U=H+D")
    assert f, r
    # 4. x of one 32-row block of a backsub_large front off by 1e-8 relative
    c = max(large, key=lambda q: int(dims[sn[1][sn[0][q]:sn[0][q + 1]]].sum()))
    idx = np.concatenate([dof[v] + np.arange(dims[v]) for v in sn[1][sn[0][c]:sn[0][c + 1]]])
    bad = dict(rd, delta=rd["delta"].copy())
    bad["delta"][idx[BLOCK:2 * BLOCK]] *= 1 + 1e-8
    f, r = fails(bad, "back_large")
    assert f, r


def test_builds_reach_the_grid():
    """On the symbolic phase alone (amalgamation on and off): every f of F_GRID, every s + 1 of S1_GRID, nn of 47 and 48
    on both sides of the first dataflow level and 49, thin dataflow fronts, a chain of three dataflow fronts, dataflow fronts
    of different shapes on one level, small leaves under dataflow fronts, and a forest."""
    seen = dict(f=set(), s1=set(), below=set(), above=set(), thin=0, chain=0, level_mix=0, small_under_df=0, forest=0)
    for name in BUILDS + ("reduced",):
        lp = front_tree(name)
        assert int(lp.var_dims.sum()) <= 1500
        for amalgamate in (True, False):
            t = supernode_table(symbolic(lp, amalgamate), lp.var_dims)
            f, s, nn, lvl, par = t["f"], t["s"], t["nn"], t["level"], t["parent"]
            df = lvl >= t["df_first"]
            if name != "reduced":
                seen["f"] |= set(f.tolist())
                seen["s1"] |= set((s + 1).tolist())
            else:   # every kernel of the emulated scenario in both modes; nn 47 / 48 below the dataflow without amalgamation
                assert (~df).any() and df.any() and backsub_large(t)
                assert amalgamate or (f.max() <= 65 and {47, 48} <= set(nn[~df].tolist()) and
                                      ((f <= THIN_F) & (nn > SMALL_MAX_N)).any())
            seen["below"] |= set(nn[~df].tolist())
            seen["above"] |= set(nn[df].tolist())
            seen["thin"] += int(((f <= THIN_F) & (nn > SMALL_MAX_N)).sum())
            seen["chain"] += sum(1 for c in range(len(par)) if df[c] and par[c] >= 0 and df[par[c]] and
                                 any(df[k] and par[k] == c for k in range(len(par))))
            seen["level_mix"] += any(len({(int(f[c]), int(s[c])) for c in np.where(df & (lvl == l))[0]}) >= 3 for l in set(lvl.tolist()))
            seen["small_under_df"] += sum(1 for c in range(len(par)) if par[c] >= 0 and nn[c] <= SMALL_MAX_N and df[par[c]]
                                          and lvl[c] == 0)
            seen["forest"] += int((par < 0).sum() >= 2)
    assert set(F_GRID) <= seen["f"], sorted(set(F_GRID) - seen["f"])
    assert set(S1_GRID) <= seen["s1"], sorted(set(S1_GRID) - seen["s1"])
    assert {47, 48} <= seen["below"] and {47, 48, 49} <= seen["above"], (sorted(seen["below"]), sorted(seen["above"]))
    for k in ("thin", "chain", "level_mix", "small_under_df", "forest"):
        assert seen[k] > 0, k
    assert front_tree("nested").hgroups


# ---- the GPU test ----------------------------------------------------------------------------------------------------------
# (amalgamation, B200_DF_MINB, B200_NO_THIN_BACKSUB) of every linear build
CONFIGS = ((True, 2, False), (True, 3, False), (False, 2, False), (False, 3, False), (True, 2, True))

SCRIPT = r"""
import os, sys, time
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import util
import test_front_shapes as T
from gtsam_b200 import capi, datasets
from oracle import oracle_py as O
ctx = capi.Context(0)
worst, strict, cells, t0 = {{}}, 0.0, 0, time.time()


def run(cell, dev, prob, sn, large, ref, f32=False):
    global cells
    for lam, diag in T.DAMPING:
        st, e0, e1, _ = dev.solve(lam, diag)
        assert st == 0, (cell, lam, diag, st)
        rd = T.readout(dev, prob)
        r, info = T.check(prob, rd, lam, diag, sn, large)
        le = abs(e1 - T.linear_error(prob, rd)) / (1e-9 * e0)
        name = "%s lam %g %s" % (cell, lam, "diag" if diag else "add")
        print(name, " ", T.fmt(r), " e1 %.3g" % le, " | strict_large %.3g cond_Rbb %.2g" % (info["strict_large"], info["cond_Rbb"]), flush=True)
        for k, v in list(r.items()) + [("e1", le)]:
            worst[k] = max(worst.get(k, 0.0), v)
        assert max(r.values()) <= 1.0 and le <= 1.0, (name, r, le)
        if lam > 0 and (lam, diag) in ref:
            rel = util.rel2(rd["delta"], ref[(lam, diag)])
            assert rel <= (1e-5 if f32 else 1e-8), (name, "delta vs oracle", rel)
        cells += 1
    return info


for name in T.BUILDS:
    lp = T.front_tree(name)
    ref = {{}}
    if name != "graded":
        orc = O.OracleLinearProblem(lp)
        for lam, diag in T.DAMPING[1:]:
            assert orc.solve(lam, diag)[0] == 0
            ref[(lam, diag)] = orc.get_delta()
        del orc
    for amalgamate, minb, no_thin in T.CONFIGS:
        with T.env(B200_NO_AMALGAMATE=None if amalgamate else "1", B200_DF_MINB=str(minb), B200_NO_THIN_BACKSUB="1" if no_thin else None):
            dev = capi.LinearDeviceProblem(ctx, lp)
        sn = dev.supernodes()
        large = T.backsub_large(T.supernode_table(sn, lp.var_dims), no_thin)
        cell = "%s %s minb %d%s" % (name, "amalg" if amalgamate else "no-amalg", minb, " no-thin" if no_thin else "")
        info = run(cell, dev, lp, sn, large, ref)
        if name == "graded":
            strict = max(strict, info["strict_large"])
        dev.close()
typed = [("sphere_tiny natural", datasets.make("sphere_tiny", layers=14, per_ring=24), False),
         ("sphere_tiny reverse", datasets.make("sphere_tiny", layers=14, per_ring=24, ordering="reverse"), False),
         ("bal_tiny bundler fp64", datasets.make("bal_tiny", ncams=40, npoints=300, camera_model="bundler"), False),
         ("bal_tiny bundler fp32", datasets.make("bal_tiny", ncams=40, npoints=300, camera_model="bundler"), True)]
for cell, prob, f32 in typed:
    orc = O.OracleProblem(prob)
    orc.set_jacobian_precision(f32)
    orc.linearize()
    ref = {{}}
    for lam, diag in T.DAMPING[1:]:
        assert orc.solve(lam, diag)[0] == 0
        ref[(lam, diag)] = orc.get_delta()
    del orc
    dev = capi.DeviceProblem(ctx, prob)
    dev.set_jacobian_precision(f32)
    dev.linearize()
    sn = dev.supernodes()
    run(cell, dev, prob, sn, T.backsub_large(T.supernode_table(sn, prob.var_dims), fused_leaf_max_f=T.LEAF_MAX_F), ref, f32)
    dev.close()
print("worst residual / bound over %d cells (%.0f s):" % (cells, time.time() - t0))
for k, v in worst.items():
    print("  %-10s %.3g" % (k, v))
print("graded build, backsub_large rows against the strict substitution bound: %.3g (not asserted)" % strict)
print("SHAPES_OK", cells)
"""


@pytest.mark.gpu
def test_front_shapes_on_gpu():
    """Every build of BUILDS on the device at every configuration of CONFIGS and every damping of DAMPING, then the typed
    problems (sphere_tiny in natural and reverse order: the generic leaves of leaf_fused_kernel; a 40-camera bal_tiny
    bundler tree in FP64 and FP32 Jacobian storage): every check of `check`, the linear error, and delta against the oracle
    on the damped, well-conditioned cells (1e-8; FP32 storage: 1e-5 with the oracle in FP32 mode).  Own process."""
    try:
        out = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT)], capture_output=True, text=True, timeout=900)
    except subprocess.TimeoutExpired:
        pytest.fail("front shapes: timed out")
    print(out.stdout)
    lines = [l for l in out.stdout.splitlines() if l.startswith("SHAPES_OK")]
    if not lines:
        pytest.fail("front shapes: did not complete: " + out.stdout[-3000:] + out.stderr[-3000:])
    assert int(lines[-1].split()[1]) > 0
