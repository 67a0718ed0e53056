"""The device marginal covariances (marginal_path_kernel, marginal_joint_kernel) on fronts wider than one CTA, long paths,
forests and point leaves, held to a componentwise forward-error bound on the device's own factor.

Both kernels run one 256-thread CTA per covariance column k and walk the clique paths of the queried variables: up,
U_P^T y = e_k (y_F = R^-T y_F, y_S -= S^T y_F), then down, U_P x = y (x_F = R^-1 (y_F - S x_S)).  U_P is U restricted to
the rows and columns of the path cliques (the union of the paths for a joint call); separators are frontals of ancestors,
so in elimination order U_P is square and upper triangular, and the covariance block is x restricted to the queried rows.

Generator: `front_tree` of tests/test_front_shapes.py on the node lists of MBUILDS.  Every claim is checked on the host-only
symbolic phase, amalgamation on and off (test_marginal_builds_reach_the_grid):
  * f in F_GRID and s in S_GRID on the path of a queried variable (every variable of a linear build is queried);
  * queried variables at the first pivot, the last pivot and pivot 256 of a 513-pivot front, and variables of a reference
    clique that amalgamation merges into its parent's supernode;
  * paths of one clique (roots) and of 13 (a chain), joint sets whose paths nest (one clique an ancestor of another's),
    a forest with joint sets spanning both trees;
  * variable dimensions 1..10 (a 10-dim variable only in joint sets), joint sets of D = 128;
  * cliques of kMargMaxF = 4096 pivots (accepted) and 4097 (rejected), compared with a float64 dense Cholesky solve;
  * "graded": the chain with every column scaled by 10^u, u in [-4, 4], so Sigma spans many orders of magnitude.
Typed problems: mixed_bal (tests/test_point_leaf_shapes.py) cal3_s2 at m_max 7 and bundler at m_max 5, every point seen
twice (an undamped factor exists), FP64 and FP32 Jacobian storage; sphere_tiny(14, 24) (dataflow fronts of nn >= 256).

Checker (`check_marginals`), in extended precision (np.longdouble) on the conditionals the device holds (`readout`): for
every column k, y = U_P^-T e_k and x = U_P^-1 y, then entry by entry
    |Sigma_hat - x| <= gamma ( |U_P^-1| |U_P| |x| + |U_P^-1| |U_P^-T| |U_P^T| |y| ),     gamma = 2 m u,  u = 2^-53.
Derivation: each entry of y (of x) is one division after a sum of at most m - 1 products, one per nonzero in its column
(row) of U_P, in whatever order and grouping the kernel uses (a separator update is a partial sum subtracted at once), so
the computed y_hat solves (U_P + dU)^T y_hat = e_k with |dU| <= gamma |U_P|, gamma = 2 m u >= gamma_m = m u / (1 - m u),
and x_hat solves (U_P + dU') x_hat = y_hat likewise.  Then x_hat - x = U_P^-1 (y_hat - y) - U_P^-1 dU' x_hat with
y_hat - y = -U_P^-T dU^T y_hat: the two terms above (to first order; the factor 2 covers the rest).  m = the most
nonzeros in a row or column of U_P, plus 1.  The bound does not assume a condition number: it is computed from U_P and
|U_P^-1| themselves (U_P^-1 in extended precision; the bound's products are sums of non-negative terms and are evaluated
in float64).  U_P^-1 is formed clique by clique from the root down, |U_P|^2 per clique: paths are kept to about 1500
dofs (MAX_PATH_DOF) so that one build checks in seconds.  Rows of U_P^-1 for a path are rows of the inverse of any larger
ancestor-closed set, so the inverse is formed once per readout over the union of the queried paths.
The chain H -> U -> Sigma is covered kernel by kernel: the same readout also goes through test_front_shapes.check at
lambda = 0 (U'U = H to a backward-error bound), and Sigma through the bound above.

test_marginal_checker_on_oracle proves the checker on the CPU oracle: it passes there, and four corruptions fail it.
test_marginal_shapes_on_gpu runs every build on the device (own process); the "marginalshapes" scenario of
tests/emu/run_scenarios.py runs a reduced build through the emulated library."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import test_front_shapes as FS
from test_point_leaf_shapes import LD, U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CTA = 256                 # threads of marginal_path_kernel / marginal_joint_kernel
MARG_MAX_F = 4096         # kMargMaxF (kernels.cuh)
MAX_D = 128               # b200_joint_marginal_covariance: scalar dimensions of one joint call
MAX_PATH_DOF = 1500
F_GRID = (1, 255, 256, 257, 512, 513)
S_GRID = (0, 255, 256, 257)
ORACLE_TOL = 1e-7         # relative to max |Sigma|, the tolerance of tests/test_gpu_marginals.py


def _r(node, *ks):
    return [(node, k) for k in ks]


# a 513-pivot root: var 0 at pivot 0, var 30 (dim 1) at pivot 255, var 31 at pivot 256, var 59 (dim 5) the last 5 pivots
ROOT513 = [1, 2] + [9] * 28 + [1] + [9] * 28 + [5]


def _chain_dims(k):
    d = k % 9 + 1
    rest = 12 - d
    return [d, 9, 9] + ([rest] if rest <= 9 else [9, rest - 9])


def mbuild_nodes(name):
    """Node lists (front_tree) of the marginal builds."""
    if name == "wide":
        # under the 513-pivot root R: fronts of f = s = 257, 256, 255, a 1-pivot leaf; a second root of 512 pivots (forest)
        return [("A", [5] + [9] * 28, _r("R", *range(2, 30), 59)), ("B", [4] + [9] * 28, _r("R", *range(0, 31))),
                ("C", [3] + [9] * 28, _r("R", *range(0, 30))), ("f1", [1], _r("R", *range(0, 31))),
                ("R", ROOT513, []), ("D", [8] + [9] * 56, [])]
    if name in ("chain", "graded"):
        # a chain c0 -> ... -> c12 of 30-pivot fronts (none amalgamated: F + S >= 48, fill > 0.15 width, not thin), every
        # dimension 1..9 and a 10-dim variable in the root; m (small, with a leaf child ml) is merged into c6 by
        # amalgamation; Q a second root
        nodes = [("ml", [2], _r("m", 0)), ("m", [4, 4], _r("c6", 0, 1))]
        chain = [("c%d" % k, _chain_dims(k), _r("c%d" % (k + 1), 0, 1, 2) if k < 11 else _r("c12", 0, 1)) for k in range(12)]
        return chain[:6] + nodes + chain[6:] + [("c12", [10, 9, 9, 2], []), ("Q", [9, 9, 9, 9, 4], [])]
    if name == "reduced":
        # the emulated scenario: a 257-pivot front with a separator of 257 under a 260-pivot root, a short chain, a forest
        return [("A", [9] * 28 + [5], _r("R", *range(0, 28), 29)), ("k0", [5, 9, 9, 9], _r("k1", 0, 1, 2)),
                ("k1", [9, 9, 9, 5], _r("k2", 0, 1, 2)), ("k2", [9, 9, 9, 9], _r("R", 0, 30)),
                ("R", [9] * 28 + [1] + [5, 2], []), ("Q", [9, 9, 3], [])]
    if name in ("big4096", "big4097"):
        return [("B", [9] * 455 + [1 if name == "big4096" else 2], [])]
    raise ValueError(name)


LINEAR = ("wide", "chain", "graded")
WELL_CONDITIONED = ("wide", "chain")


def mbuild(name):
    return FS.front_tree(name, nodes=mbuild_nodes(name), graded=name == "graded")


def var_of_node(name):
    """{(node, k): variable id} of a build."""
    out, v = {}, 0
    for node, vd, _ in mbuild_nodes(name):
        for k in range(len(vd)):
            out[(node, k)] = v
            v += 1
    return out


def joint_sets(name):
    """Joint queries of a linear build (ascending ids, the order of the result's blocks): nested paths, forest-spanning
    sets, D = 128, a 10-dim variable."""
    return [tuple(sorted(vs)) for vs in _joint_sets(name)]


def _joint_sets(name):
    V = var_of_node(name)
    if name == "wide":
        return [(V["R", 0], V["R", 31], V["R", 59]),                       # first pivot, pivot 256, last pivot
                (V["A", 0], V["A", 28], V["R", 31]),                      # A's clique is a child of R's: nested paths
                (V["A", 3], V["D", 0], V["D", 56]),                       # both trees
                (V["f1", 0], V["B", 0], V["C", 28], V["D", 30]),
                tuple([V["R", 0], V["R", 30]] + [V["R", k] for k in range(2, 16)])]     # D = 1 + 1 + 14 * 9 = 128
    if name == "reduced":
        return [(V["A", 0], V["R", 28], V["R", 30]), (V["k0", 0], V["k2", 3], V["Q", 1]), (V["A", 28], V["Q", 0])]
    return [(V["c0", 0], V["c5", 1], V["c12", 0]),                        # 13-deep path nested in the root's; 10-dim var
            (V["c0", 1], V["Q", 2]),                                      # both trees
            (V["ml", 0], V["m", 1], V["c6", 2], V["c12", 3]),             # through the merged clique
            (V["c3", 0], V["c3", 2], V["c9", 1], V["Q", 4])]


def var_clique(cliques, nvars):
    fp, fv, _, _, par = cliques
    vc = np.full(nvars, -1, dtype=np.int64)
    for c in range(len(par)):
        vc[fv[fp[c]:fp[c + 1]]] = c
    return vc


def path_of(cliques, vc, vs):
    """Ascending clique ids of the union of the paths of variables vs (what b200_joint_marginal_covariance walks)."""
    par = cliques[4]
    on = set()
    for v in vs:
        c = int(vc[v])
        while c >= 0 and c not in on:
            on.add(c)
            c = int(par[c])
    return sorted(on)


def path_dofs(prob, cliques, path):
    fp, fv = cliques[0], cliques[1]
    dims, dof = prob.var_dims, prob.dof_offsets()
    return sum(int(dims[fv[fp[c]:fp[c + 1]]].sum()) for c in path)


class Factor:
    """The conditionals of a readout as one upper-triangular U in elimination order, with U^-1 (longdouble) formed from the
    root down over the union of the cliques of `need` (variables)."""

    def __init__(self, prob, rd, need):
        self.prob = prob
        fp, fv, sp, sv, par = self.cl = rd["cliques"]
        dims, dof = prob.var_dims, prob.dof_offsets()
        self.vc = var_clique(self.cl, prob.nvars)
        cls = path_of(self.cl, self.vc, need)
        self.cols = {}
        pos = {}                                     # dof -> index in the union, in elimination order
        for c in cls:
            for v in fv[fp[c]:fp[c + 1]]:
                for q in range(dof[v], dof[v] + dims[v]):
                    pos[int(q)] = len(pos)
        self.pos = pos
        n = self.n = len(pos)
        self.U = np.zeros((n, n), dtype=LD)
        self.Ui = np.zeros((n, n), dtype=LD)
        idx = lambda vs: np.array([pos[int(q)] for v in vs for q in range(dof[v], dof[v] + dims[v])], dtype=np.int64)
        pcols = {}
        for c in reversed(cls):                      # parents have larger ids: the root first
            fr, se = idx(fv[fp[c]:fp[c + 1]]), idx(sv[sp[c]:sp[c + 1]])
            cd = rd["conds"][c].astype(LD)
            f = len(fr)
            R, S = cd[:, :f], cd[:, f:-1]
            self.U[np.ix_(fr, fr)] = R
            self.U[np.ix_(fr, se)] = S
            P = np.concatenate([fr, pcols[int(par[c])]]) if par[c] >= 0 else fr
            pcols[c] = P
            rhs = np.zeros((f, len(P)), dtype=LD)
            rhs[:, :f] = np.eye(f, dtype=LD)
            if len(se):
                rhs -= S @ self.Ui[np.ix_(se, P)]
            self.Ui[np.ix_(fr, P)] = FS._tri_inv(R) @ rhs
        self.aU = np.abs(self.U).astype(np.float64)
        self.aUi = np.abs(self.Ui).astype(np.float64)
        self.Ui64 = self.Ui.astype(np.float64)
        self.idx = idx

    def reference(self, vs):
        """Sigma of variables vs (ascending) in extended precision: rows Q of U^-1 U^-T."""
        Q = self.idx(vs)
        return self.Ui[Q] @ self.Ui[Q].T

    def ratio(self, vs, S):
        """max |S - Sigma| / bound over the entries of S (module docstring)."""
        Q = self.idx(vs)
        P = self.idx([v for c in path_of(self.cl, self.vc, vs) for v in self.cl[1][self.cl[0][c]:self.cl[0][c + 1]]])
        aU, Ui = self.aU[np.ix_(P, P)], self.Ui64[np.ix_(P, P)]
        aUi = self.aUi[np.ix_(P, P)]
        m = int(max((aU != 0).sum(0).max(), (aU != 0).sum(1).max())) + 1
        Y = self.Ui64[np.ix_(Q, P)].T                # column k: y = U_P^-T e_k
        X = Ui @ Y
        aUiQ = self.aUi[np.ix_(Q, P)]
        bound = 2 * m * U * (aUiQ @ (aU @ np.abs(X)) + aUiQ @ (aUi.T @ (aU.T @ np.abs(Y))))
        res = np.abs(np.asarray(S, dtype=LD) - self.reference(vs)).astype(np.float64)
        if np.any((bound == 0) & (res != 0)):
            return np.inf
        nz = bound > 0
        return float((res[nz] / bound[nz]).max()) if nz.any() else 0.0


def check_marginals(prob, rd, singles, joints):
    """(worst ratio of the single-variable marginals, of the joint marginals): singles {var: Sigma}, joints [(vars,
    Sigma)]; <= 1 passes."""
    need = list(singles) + [v for vs, _ in joints for v in vs]
    F = Factor(prob, rd, need)
    rs = max((F.ratio([v], S) for v, S in singles.items()), default=0.0)
    rj = max((F.ratio(list(vs), S) for vs, S in joints), default=0.0)
    return rs, rj


def walk(prob, rd, vs, skip_sep=None, skip_pivot=None):
    """A float64 numpy copy of marginal_joint_kernel on the readout's cliques; skip_sep: a clique whose separator update is
    left out; skip_pivot: (clique, i) -- the forward solve never updates y_i of that clique (what a thread-stride loop that
    stops after its first pass does to entry 256)."""
    fp, fv, sp, sv, par = rd["cliques"]
    dims, dof = prob.var_dims, prob.dof_offsets()
    vc = var_clique(rd["cliques"], prob.nvars)
    path = path_of(rd["cliques"], vc, vs)
    cols = lambda us: np.concatenate([dof[u] + np.arange(dims[u]) for u in us]) if len(us) else np.zeros(0, np.int64)
    dofs = cols(vs)
    out = np.zeros((len(dofs), len(dofs)))
    for k, dk in enumerate(dofs):
        w = np.zeros(int(dof[-1]))
        w[dk] = 1.0
        for c in path:
            di = cols(list(fv[fp[c]:fp[c + 1]]) + list(sv[sp[c]:sp[c + 1]]))
            M = rd["conds"][c]
            f = M.shape[0]
            y = w[di[:f]].copy()
            for i in range(f):
                y[i] /= M[i, i]
                upd = M[i, i + 1:f] * y[i]
                if skip_pivot is not None and skip_pivot[0] == c and i < skip_pivot[1]:
                    upd[skip_pivot[1] - i - 1] = 0.0
                y[i + 1:] -= upd
            w[di[:f]] = y
            if c != skip_sep:
                w[di[f:]] -= M[:, f:-1].T @ y
        for c in reversed(path):
            di = cols(list(fv[fp[c]:fp[c + 1]]) + list(sv[sp[c]:sp[c + 1]]))
            M = rd["conds"][c]
            f = M.shape[0]
            y = w[di[:f]] - M[:, f:-1] @ w[di[f:]]
            for i in range(f - 1, -1, -1):
                y[i] /= M[i, i]
                y[:i] -= M[:i, i] * y[i]
            w[di[:f]] = y
        out[:, k] = w[dofs]
    return out


def queried(prob):
    """Variables a single-variable call accepts (d <= 9)."""
    return [v for v in range(prob.nvars) if prob.var_dims[v] <= 9]


# ---- shapes, on the symbolic phase ---------------------------------------------------------------------------------------
def _supernodes(lp, amalgamate):
    from gtsam_b200 import capi
    with FS.env(B200_NO_AMALGAMATE=None if amalgamate else "1"):
        return capi.linear_symbolic(lp, with_slots=True)[:5], capi.linear_symbolic(lp)


def test_marginal_builds_reach_the_grid():
    """On the symbolic phase alone (amalgamation on and off): every f of F_GRID and s of S_GRID on a queried path, the
    placement of queried variables (first pivot, last pivot, pivot 256 of a front wider than 256, a merged reference
    clique), paths of 1 and >= 12 supernodes, nested joint paths, forests with spanning joint sets, dimensions 1..10,
    D = 128 joint sets, 4096- and 4097-pivot cliques, and paths within MAX_PATH_DOF."""
    for amalgamate in (True, False):
        seen = dict(f=set(), s=set(), dims=set(), first=0, last=0, p256=0, merged=0, depth1=0, depth12=0, nested=0,
                    forest=0, d128=0)
        for name in LINEAR + ("reduced",):
            lp = mbuild(name)
            sn, ref = _supernodes(lp, amalgamate)
            fp, fv, sp, sv, par = sn
            dims, dof = lp.var_dims, lp.dof_offsets()
            t = FS.supernode_table(sn, dims)
            vc = var_clique(sn, lp.nvars)
            depth = np.zeros(len(par), dtype=np.int64)
            for c in range(len(par) - 1, -1, -1):
                depth[c] = 1 + (depth[par[c]] if par[c] >= 0 else 0)
            seen["dims"] |= set(dims.tolist())
            for v in range(lp.nvars):
                c = vc[v]
                front = [int(u) for u in fv[fp[c]:fp[c + 1]]]
                slot = int(sum(dims[u] for u in front[:front.index(v)]))
                seen["first"] += slot == 0 and t["f"][c] > CTA
                seen["last"] += slot + dims[v] == t["f"][c] and t["f"][c] > CTA
                seen["p256"] += slot == CTA and t["f"][c] > CTA
                pc = path_of(sn, vc, [v])
                assert path_dofs(lp, sn, pc) <= MAX_PATH_DOF
                if name != "reduced":
                    seen["f"] |= {int(t["f"][q]) for q in pc}
                    seen["s"] |= {int(t["s"][q]) for q in pc}
                seen["depth1"] += len(pc) == 1
                seen["depth12"] += len(pc) >= 12
            # a reference clique merged into a bigger supernode, its variables not first in the front
            rvc = var_clique(ref, lp.nvars)
            for v in range(lp.nvars):
                c, r = vc[v], rvc[v]
                merged = set(fv[fp[c]:fp[c + 1]].tolist()) != set(ref[1][ref[0][r]:ref[0][r + 1]].tolist())
                seen["merged"] += bool(merged) and int(fv[fp[c]]) != v
            for vs in joint_sets(name):
                roots = set()
                for v in vs:
                    c = int(vc[v])
                    while par[c] >= 0:
                        c = int(par[c])
                    roots.add(c)
                seen["forest"] += len(roots) >= 2
                anc = [set(path_of(sn, vc, [v])) for v in vs]
                seen["nested"] += any(vc[w] in anc[a] and vc[u] != vc[w] for a, u in enumerate(vs) for w in vs)
                seen["d128"] += int(dims[list(vs)].sum()) == MAX_D
        assert set(F_GRID) <= seen["f"], (amalgamate, sorted(seen["f"]))
        assert set(S_GRID) <= seen["s"], (amalgamate, sorted(seen["s"]))
        assert set(range(1, 11)) <= seen["dims"]
        for k in ("first", "last", "p256", "depth1", "depth12", "nested", "forest", "d128"):
            assert seen[k] > 0, (amalgamate, k)
        assert seen["merged"] > 0 or not amalgamate
    # wide fronts cross the CTA's thread count; the 4096 / 4097 cliques straddle kMargMaxF
    for name, f in (("big4096", MARG_MAX_F), ("big4097", MARG_MAX_F + 1)):
        t = FS.supernode_table(_supernodes(mbuild(name), True)[0], mbuild(name).var_dims)
        assert t["f"].tolist() == [f]


# ---- the checker proven on the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", LINEAR)
def test_marginal_checker_on_oracle(name):
    """The checker passes on the CPU oracle's factor and marginals (every variable, every joint set), the same readout
    passes test_front_shapes.check at lambda = 0, and four corruptions each fail the checker."""
    from oracle import oracle_py as O
    lp = mbuild(name)
    orc = O.OracleLinearProblem(lp)
    qv = queried(lp)
    st, full = orc.joint_marginal_covariance(range(lp.nvars))      # one solve: every diagonal block
    assert st == 0
    dof = lp.dof_offsets()
    singles = {v: full[dof[v]:dof[v + 1], dof[v]:dof[v + 1]] for v in qv}
    V = var_of_node(name)
    probe = [V["R", 31], V["R", 0]] if name == "wide" else [V["c0", 0], V["ml", 0]]
    for v in probe:                                                 # the single-variable call gives the same blocks
        st, S = orc.marginal_covariance(v)
        assert st == 0 and np.abs(S - singles[v]).max() <= 1e-12 * np.abs(S).max()
    joints = []
    for vs in joint_sets(name):
        st, S = orc.joint_marginal_covariance(vs)
        assert st == 0
        joints.append((vs, S))
    rd = FS.readout(orc, lp)
    sn = FS.symbolic(lp)
    r, _ = FS.check(lp, rd, 0.0, False, sn, FS.backsub_large(FS.supernode_table(sn, lp.var_dims)))
    assert max(r.values()) <= 1.0, r
    F = Factor(lp, rd, list(range(lp.nvars)))
    rs = max(F.ratio([v], S) for v, S in singles.items())
    rj = max(F.ratio(list(vs), S) for vs, S in joints)
    print(name, FS.fmt(r), " single %.3g joint %.3g" % (rs, rj))
    assert rs <= 1.0 and rj <= 1.0, (rs, rj)
    # the numpy walk (the kernel's algorithm) passes too
    wv = V["R", 0] if name == "wide" else V["c0", 0]
    assert F.ratio([wv], walk(lp, rd, [wv])) <= 1.0
    # 1. one entry in a column of pivot >= 256 (the diagonal of R's variable at pivot 256), off by 1e-8 relative;
    #    on the chain builds, the last variable of the root
    v = V["R", 31] if name == "wide" else V["c12", 3]
    S = singles[v].copy()
    S[0, 0] *= 1 + 1e-8
    assert F.ratio([v], S) > 1.0
    # 2. the walk without one clique's separator update (the queried variable's own clique)
    vc = F.vc
    v = V["A", 0] if name == "wide" else V["c0", 0]
    assert F.ratio([v], walk(lp, rd, [v], skip_sep=int(vc[v]))) > 1.0
    # 3. the forward solve never updates entry 256 of a front wider than 256 (the wide build; on the chain builds, entry
    #    16 of the variable's own 30-pivot clique)
    if name == "wide":
        v, c, i = V["R", 0], int(vc[V["R", 0]]), CTA
    else:
        v = V["c0", 0]
        c, i = int(vc[v]), 16
    assert F.ratio([v], walk(lp, rd, [v], skip_pivot=(c, i))) > 1.0
    # 4. two variables' blocks of a joint result swapped out of sorted-key order
    vs, S = joints[0]
    d = [int(lp.var_dims[u]) for u in vs]
    o = np.concatenate([[0], np.cumsum(d)])
    perm = np.concatenate([np.arange(o[1], o[2]), np.arange(o[0], o[1]), np.arange(o[2], o[-1])])
    assert F.ratio(list(vs), S[np.ix_(perm, perm)]) > 1.0


# ---- the GPU test ----------------------------------------------------------------------------------------------------------
# (amalgamation, B200_DF_MINB) of every build
CONFIGS = ((True, 2), (True, 3), (False, 2), (False, 3))

SCRIPT = r"""
import os, sys, time, copy
import ctypes as C
import numpy as np
import scipy.linalg as sl
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import util
import test_marginal_shapes as T
import test_front_shapes as FS
import test_point_leaf_shapes as PL
from gtsam_b200 import capi, datasets, problem as P
from oracle import oracle_py as O
ctx = capi.Context(0)
worst, cells, t0 = {{}}, 0, time.time()
bitwise = dict(joint_diag=0, repeat=0, cross_zero=0)


def note(key, v):
    worst[key] = max(worst.get(key, 0.0), v)


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max())


def run_cell(cell, dev, prob, qv, sets, ref, tag, f32=False):
    # singles first (they run the undamped factorisation), then the readout of that factor, then the joints
    global cells
    singles = {{v: dev.marginal_covariance(v) for v in qv}}
    rd = FS.readout(dev, prob)
    joints = [(vs, dev.joint_marginal_covariance(vs)) for vs in sets]
    # the factor: U'U = H (backward error), on the same readout
    if getattr(prob, "name", "").startswith("mixed_bal"):
        r = PL.check(prob, rd, 0.0, False)
    else:
        sn = dev.supernodes()
        r, _ = FS.check(prob, rd, 0.0, False, sn, FS.backsub_large(FS.supernode_table(sn, prob.var_dims),
                        fused_leaf_max_f=0 if isinstance(prob, FS.LN.LinearProblem) else FS.LEAF_MAX_F))
    rs, rj = T.check_marginals(prob, rd, singles, joints)
    print("%-40s factor %.3g  single %.3g  joint %.3g" % (cell, max(r.values()), rs, rj), flush=True)
    note(tag + " factor", max(r.values())); note(tag + " single", rs); note(tag + " joint", rj)
    assert max(r.values()) <= 1.0 and rs <= 1.0 and rj <= 1.0, (cell, r, rs, rj)
    # invariants: joint diagonal blocks = the single marginals bit for bit; cross-tree blocks exactly zero
    vc = T.var_clique(rd["cliques"], prob.nvars)
    par = rd["cliques"][4]
    def root(v):
        c = int(vc[v])
        while par[c] >= 0:
            c = int(par[c])
        return c
    for vs, S in joints:
        o = np.concatenate([[0], np.cumsum([int(prob.var_dims[u]) for u in vs])])
        for a, u in enumerate(vs):
            if u in singles:
                assert np.array_equal(S[o[a]:o[a + 1], o[a]:o[a + 1]], singles[u]), (cell, vs, u, "joint diagonal != single")
                bitwise["joint_diag"] += 1
            for b, w in enumerate(vs):
                if root(u) != root(w):
                    assert np.all(S[o[a]:o[a + 1], o[b]:o[b + 1]] == 0.0), (cell, vs, u, w, "cross-tree block")
                    bitwise["cross_zero"] += 1
    # the same variable again (a front wider than the CTA where there is one): bit-identical
    v = max(qv, key=lambda u: rd["conds"][int(vc[u])].shape[0])
    assert np.array_equal(dev.marginal_covariance(v), singles[v]), (cell, v, "repeat")
    bitwise["repeat"] += 1
    if ref is not None:
        rs_ref, rj_ref = ref
        d = max([rel(singles[v], rs_ref[v]) for v in qv] + [rel(S, R) for (_, S), R in zip(joints, rj_ref)])
        print("%-40s vs oracle %.3g" % (cell, d), flush=True)
        note(tag + " vs oracle", d)
        assert d <= T.ORACLE_TOL, (cell, "vs oracle", d)
    cells += 1


def oracle_ref(orc, qv, sets):
    # the single marginals are the diagonal blocks of one joint call over all of them (one factorisation)
    st, S = orc.joint_marginal_covariance(qv)
    assert st == 0
    o = np.concatenate([[0], np.cumsum([int(orc.prob.var_dims[v]) for v in sorted(qv)])])
    rs = {{v: S[o[a]:o[a + 1], o[a]:o[a + 1]] for a, v in enumerate(sorted(qv))}}
    rj = []
    for vs in sets:
        st, S = orc.joint_marginal_covariance(vs)
        assert st == 0
        rj.append(S)
    return rs, rj


# ---- linear builds
for name in T.LINEAR:
    lp = T.mbuild(name)
    qv, sets = T.queried(lp), T.joint_sets(name)
    ref = oracle_ref(O.OracleLinearProblem(lp), qv, sets) if name in T.WELL_CONDITIONED else None
    for amalgamate, minb in T.CONFIGS:
        with FS.env(B200_NO_AMALGAMATE=None if amalgamate else "1", B200_DF_MINB=str(minb)):
            dev = capi.LinearDeviceProblem(ctx, lp)
        run_cell("%s %s minb %d" % (name, "amalg" if amalgamate else "no-amalg", minb), dev, lp, qv, sets, ref,
                 "graded" if name == "graded" else "linear")
        dev.close()

# ---- typed problems
typed = []
for model, m_max in (("cal3_s2", 7), ("bundler", 5)):
    prob = PL.mixed_bal(model, m_max, m_min=2)
    typed += [("%s m%d fp64" % (model, m_max), prob, False), ("%s m%d fp32" % (model, m_max), prob, True)]
sphere = datasets.make("sphere_tiny", layers=14, per_ring=24)
typed.append(("sphere_tiny 14x24", sphere, False))
for cell, prob, f32 in typed:
    dev = capi.DeviceProblem(ctx, prob)
    dev.set_jacobian_precision(f32)
    cl = dev.cliques()
    vc = T.var_clique(cl, prob.nvars)
    if getattr(prob, "name", "").startswith("mixed_bal"):
        cams = [v for v in range(prob.nvars) if prob.var_type[v] != P.VAR_POINT3]
        pts = [v for v in range(prob.nvars) if prob.var_type[v] == P.VAR_POINT3 and cl[4][vc[v]] >= 0]
        width = lambda v: int(cl[2][vc[v] + 1] - cl[2][vc[v]])
        pts = sorted(pts, key=lambda v: (width(v), v))
        picks = [pts[int(i)] for i in np.linspace(0, len(pts) - 1, 40)]
        qv = cams + picks
        g = prob.groups[0]
        sets = []
        for p in (picks[0], picks[20], picks[-1]):
            cs = sorted(set(g.keys[g.keys[:, 1] == p, 0].tolist()))
            if 3 + sum(int(prob.var_dims[c]) for c in cs) <= 128:          # (the widest off-path points see 20 cameras)
                sets.append(tuple(sorted(cs + [p])))
        assert sets
    else:
        # every 8th pose whose path stays within MAX_PATH_DOF, and pairs of them
        qv = [v for v in range(0, prob.nvars, 8) if T.path_dofs(prob, cl, T.path_of(cl, vc, [v])) <= T.MAX_PATH_DOF]
        sets = [tuple(qv[i:i + 3]) for i in range(0, min(len(qv), 12), 3)]
    orc = O.OracleProblem(prob)
    orc.set_jacobian_precision(f32)
    ref = oracle_ref(orc, qv, sets)
    del orc
    run_cell(cell, dev, prob, qv, sets, ref, "typed")
    dev.close()

# ---- kMargMaxF: 4096 pivots accepted (against a dense float64 Cholesky solve), 4097 rejected
for name in ("big4096", "big4097"):
    lp = T.mbuild(name)
    dev = capi.LinearDeviceProblem(ctx, lp)
    last = lp.nvars - 1
    if name == "big4097":
        for call in (lambda: dev.marginal_covariance(0), lambda: dev.joint_marginal_covariance([0, last])):
            try:
                call()
                raise AssertionError("4097 pivots accepted")
            except capi.B200Error as e:
                assert e.code == P.INVALID_ARGUMENT and "more than 4096 pivots" in str(e), e
        print("big4097: rejected with B200_INVALID_ARGUMENT", flush=True)
    else:
        n = int(lp.dof_offsets()[-1])
        H = np.zeros((n, n))
        dof = lp.dof_offsets()
        J = [dev.get_jacobians(gi) for gi in range(len(lp.groups))]
        for g, Jg in zip(lp.groups, J):
            for k in range(g.count):
                cols = np.concatenate([dof[v] + np.arange(lp.var_dims[v]) for v in g.keys[k]])
                A = Jg[k][:, :-1]
                H[np.ix_(cols, cols)] += A.T @ A
        cf = sl.cho_factor(H)
        d = 0.0
        for v in (0, 28, 29, last):
            cols = np.arange(dof[v], dof[v + 1])
            E = np.zeros((n, len(cols))); E[cols, np.arange(len(cols))] = 1
            d = max(d, rel(dev.marginal_covariance(v), sl.cho_solve(cf, E)[cols]))
        vs = (0, 29, last)
        cols = np.concatenate([np.arange(dof[v], dof[v + 1]) for v in vs])
        E = np.zeros((n, len(cols))); E[cols, np.arange(len(cols))] = 1
        d = max(d, rel(dev.joint_marginal_covariance(vs), sl.cho_solve(cf, E)[cols]))
        print("big4096: vs float64 cho_solve %.3g" % d, flush=True)
        note("4096 vs cho_solve", d)
        assert d <= 1e-8, d
    dev.close()

# ---- argument errors
lp = T.mbuild("chain")
dev = capi.LinearDeviceProblem(ctx, lp)
V = T.var_of_node("chain")
L, h = dev.L, dev.h
def status_single(v):
    out = np.zeros(100)
    return L.b200_marginal_covariance(h, int(v), out.ctypes.data_as(C.POINTER(C.c_double)))
def status_joint(vs):
    vs = np.array(vs, dtype=np.int64)
    out = np.zeros(200 * 200)
    return L.b200_joint_marginal_covariance(h, vs.ctypes.data_as(C.POINTER(C.c_int64)), len(vs), out.ctypes.data_as(C.POINTER(C.c_double)))
assert status_single(-1) == P.INVALID_ARGUMENT and status_single(lp.nvars) == P.INVALID_ARGUMENT
assert status_single(V["c12", 0]) == P.INVALID_ARGUMENT                     # d = 10
assert "dimension > 9" in L.b200_last_error_string().decode()
assert status_joint([V["c12", 0], V["c0", 0]]) == P.INVALID_ARGUMENT       # not ascending
assert status_joint([V["c0", 0], V["c0", 0]]) == P.INVALID_ARGUMENT        # duplicate
assert status_joint([V["c0", 0], lp.nvars]) == P.INVALID_ARGUMENT          # out of range
assert "ascending" in L.b200_last_error_string().decode()
assert status_joint([V["c0", 0], V["c12", 0]]) == 0                        # the 10-dim variable in a joint
dev.close()
wl = T.mbuild("wide")
dev = capi.LinearDeviceProblem(ctx, wl)
L, h = dev.L, dev.h
W = T.var_of_node("wide")
d128 = T.joint_sets("wide")[-1]
assert int(wl.var_dims[list(d128)].sum()) == 128 and status_joint(list(d128)) == 0
d129 = sorted(set(d128) - {{W["R", 30]}} | {{W["R", 1]}})
assert int(wl.var_dims[d129].sum()) == 129 and status_joint(d129) == P.INVALID_ARGUMENT
assert "more than 128" in L.b200_last_error_string().decode()
dev.close()
print("argument errors: out of range, not ascending, duplicate, d = 10, D = 129, 4097 pivots rejected", flush=True)

# ---- mutators: after each one the next marginal describes the new state
def compare(what, dev, orc, prob, vs, prev, moved=True):
    S = dev.joint_marginal_covariance(vs)
    st, R = orc.joint_marginal_covariance(vs)
    assert st == 0
    if moved:
        m = rel(R, prev)
        assert m >= 1e-3, (what, "oracle Sigma moved only", m)
    d = rel(S, R)
    rd = FS.readout(dev, prob)
    rs, rj = T.check_marginals(prob, rd, {{}}, [(vs, S)])
    print("mutator %-28s vs oracle %.3g  checker %.3g" % (what, d, rj), flush=True)
    note("mutator vs oracle", d); note("mutator checker", rj)
    assert d <= T.ORACLE_TOL and rj <= 1.0, (what, d, rj)
    return R

# linear: linear_update, linear_update_hessian, a damped solve, a failed solve
lp = FS.front_tree("nested")
dev, orc = capi.LinearDeviceProblem(ctx, lp), O.OracleLinearProblem(lp)
vs = (0, 3, 12, lp.nvars - 1)       # l1, l4, the HessianFactor's M2, the root
R = compare("initial", dev, orc, lp, vs, None, moved=False)
g0 = lp.groups[0]
Ab = np.ascontiguousarray(np.transpose(dev.get_jacobians(0), (0, 2, 1))) * 1.5
dev.update(0, Ab); orc.update(0, Ab)
R = compare("linear_update", dev, orc, lp, vs, R)
hg = lp.hgroups[0]
info = hg.info * 2.0
dev.update_hessian(0, info); orc.update_hessian(0, info)
R = compare("linear_update_hessian", dev, orc, lp, vs, R)
dev.solve(10.0)
R = compare("damped solve", dev, orc, lp, vs, R, moved=False)
# a leaf variable loses its only factor: indeterminate; restored: the next marginal succeeds
leaf = next(gi for gi, g in enumerate(lp.groups) if g.keys[0][0] == 0)
Ab = np.ascontiguousarray(np.transpose(dev.get_jacobians(leaf), (0, 2, 1)))
dev.update(leaf, np.zeros_like(Ab))
try:
    dev.marginal_covariance(0)
    raise AssertionError("indeterminate system not reported")
except capi.IndeterminantLinearSystemException:
    pass
dev.update(leaf, Ab)
R = compare("failed solve, then fixed", dev, orc, lp, vs, R, moved=False)
dev.close(); del orc

# typed: set_values, set_values_view, accept_step, restore_values, set_group_noise, set_jacobian_precision, an LM try,
# a Dogleg step
from gtsam_b200 import optimizer
prob = datasets.make("sphere_tiny")
dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
vs = (0, 7, prob.nvars - 1)
v0 = dev.get_values()
orc.linearize(); assert orc.solve(1e-3)[0] == 0; orc.try_step(); orc.accept_step()
v1 = orc.get_values()
orc.set_values(v0)
R = compare("initial", dev, orc, prob, vs, None, moved=False)
dev.set_values(v1); orc.set_values(v1)
R = compare("set_values", dev, orc, prob, vs, R)
dev.set_values_view(np.ascontiguousarray(v0[dev.view_index(0)])); orc.set_values(v0)
R = compare("set_values_view", dev, orc, prob, vs, R)
dev.save_values()
dev.linearize(); assert dev.solve(1e-3)[0] == 0; dev.try_step(); dev.accept_step()
orc.set_values(dev.get_values())
R = compare("accept_step", dev, orc, prob, vs, R)
dev.restore_values(); orc.set_values(v0)
R = compare("restore_values", dev, orc, prob, vs, R)
gi = 0
g = prob.groups[gi]
noisy = copy.deepcopy(prob)
noisy.groups[gi] = copy.deepcopy(g)
noisy.groups[gi].noise = np.asarray(g.noise, dtype=np.float64) * 3.0
dev.set_group_noise(gi, g.noise_kind, noisy.groups[gi].noise)
orc = O.OracleProblem(noisy); orc.set_values(v0)
R = compare("set_group_noise", dev, orc, prob, vs, R)
dev.set_jacobian_precision(True); orc.set_jacobian_precision(True)
before = dev.joint_marginal_covariance(vs)
R = compare("set_jacobian_precision", dev, orc, prob, vs, R, moved=False)
dev.set_jacobian_precision(False); orc.set_jacobian_precision(False)
dev.linearize(); assert dev.solve(10.0)[0] == 0; dev.try_step()
R = compare("LM try", dev, orc, prob, vs, R, moved=False)
dl = optimizer.DoglegOptimizer(ctx, noisy, device_problem=dev)
dl.iterate()
orc.set_values(dev.get_values())
R = compare("Dogleg step", dev, orc, prob, vs, R)
dev.close()

print("worst ratio over %d cells (%.0f s):" % (cells, time.time() - t0))
for k, v in worst.items():
    print("  %-22s %.3g" % (k, v))
print("bitwise: %(joint_diag)d joint diagonal blocks, %(repeat)d repeats, %(cross_zero)d cross-tree blocks" % bitwise)
print("MARGINAL_SHAPES_OK", cells)
"""


@pytest.mark.gpu
def test_marginal_shapes_on_gpu():
    """Every linear build at every configuration of CONFIGS (every single-variable marginal, every joint set), the typed
    problems (FP64 and FP32 storage), the kMargMaxF guard, the argument errors and the mutator walk; the checker, the
    backward-error check of the factor, the oracle on the well-conditioned builds, and the bitwise invariants (joint
    diagonal blocks = single marginals, cross-tree blocks = 0, a repeated query).  Own process."""
    try:
        out = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT)], capture_output=True, text=True, timeout=1200)
    except subprocess.TimeoutExpired:
        pytest.fail("marginal shapes: timed out")
    print(out.stdout)
    lines = [l for l in out.stdout.splitlines() if l.startswith("MARGINAL_SHAPES_OK")]
    if not lines:
        pytest.fail("marginal shapes: did not complete: " + out.stdout[-3000:] + out.stderr[-3000:])
    assert int(lines[-1].split()[1]) > 0
