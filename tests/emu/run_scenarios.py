"""Scenarios run against the HOST-EMULATION build of the whole library (tests/test_library_emulation.py starts this file
in its own process: `python run_scenarios.py <libgtsam_b200_emu.so> <scenario>...`).  TEST INFRASTRUCTURE."""
import os
import sys
import time

os.environ["B200_NO_GRAPH"] = "1"      # CUDA graphs are not emulated: eager launches
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gtsam_b200 import capi  # noqa: E402

capi.LIB_PATH = sys.argv[1]
import numpy as np  # noqa: E402
import util  # noqa: E402
from gtsam_b200 import linear as LN, optimizer, problem as P  # noqa: E402
from oracle import oracle_py as O  # noqa: E402

ctx = capi.Context(0)


def typed(case):
    prob = util.load_case(case)
    for kind, lam, diag in (("dump0", 0.0, 0), ("dump1", 1e-2, 1)):
        dev = capi.DeviceProblem(ctx, prob)
        util.check_against_dump(dev, prob, util.golden(case, kind), lam, diag)
        dev.close()
    # gradientAtZero = -A'b of the whitened blocks (which the dumps above pinned on the reference)
    dev = capi.DeviceProblem(ctx, prob)
    dev.linearize()
    off = prob.dof_offsets()
    g = np.zeros(off[-1])
    for gi, grp in enumerate(prob.groups):
        J = dev.get_jacobians(gi)                  # (count, rows, ncols)
        contrib = -np.einsum("frc,fr->fc", J[:, :, :-1], J[:, :, -1])
        col = 0
        for a in range(grp.keys.shape[1]):
            d = int(prob.var_dims[grp.keys[0, a]]) if grp.count else 0
            np.add.at(g, off[grp.keys[:, a]][:, None] + np.arange(d)[None, :], contrib[:, col:col + d])
            col += d
    assert util.relmax(dev.gradient_at_zero(), g) <= 1e-12
    dev.close()
    # LM to convergence: same error / lambda sequence as the reference
    ref = util.golden(case, "lm")
    prm = optimizer.LevenbergMarquardtParams.CeresDefaults() if case in util.CERES_CASES else optimizer.LevenbergMarquardtParams()
    lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, prm)
    errs = [lm.error()]
    for _ in range(len(ref["lm_errors"]) - 1):
        lm.iterate()
        errs.append(lm.error())
    # (dubrovnik-3-7: cond(H) ~ 1e15 at the first lambdas -> trajectories agree to ~1e-6 only, as in tests/test_oracle_golden.py)
    assert np.allclose(errs, ref["lm_errors"], rtol=1e-5 if case.startswith("dub") else 1e-7, atol=1e-10), (errs, ref["lm_errors"])
    assert abs(lm.lambda_() - ref["lm_lambdas"][-1]) <= 1e-12 * ref["lm_lambdas"][-1]


def fp32(case):
    prob = util.load_case(case)
    ref = util.golden(case, "dump0")
    dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
    dev.linearize()
    st64 = dev.solve(0.0)[0]
    d64, j64 = dev.get_delta(), dev.get_jacobians(0)
    dev.set_jacobian_precision(True); orc.set_jacobian_precision(True)
    dev.linearize(); orc.linearize()
    for gi in range(len(prob.groups)):
        J = dev.get_jacobians(gi)
        assert np.array_equal(J, J.astype(np.float32).astype(np.float64))
        assert util.relmax(J, orc.get_jacobians(gi)) <= 1e-6 and util.relmax(J, util.ref_jacobians(prob, ref, gi)) <= 1e-6
    assert util.relmax(dev.hessian_diagonal(), orc.hessian_diagonal()) <= 1e-6
    st, e0, e1, _ = dev.solve(1e-2, True)
    so, f0, f1, _ = orc.solve(1e-2, True)
    assert st == so == 0 and util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-5
    assert abs(e0 - f0) <= 1e-6 * f0 and abs(e1 - f1) <= 1e-5 * f0
    dev.set_jacobian_precision(False)
    dev.linearize()
    assert dev.solve(0.0)[0] == st64 and np.array_equal(dev.get_jacobians(0), j64)
    assert st64 != 0 or util.rel2(dev.get_delta(), d64) <= 1e-10     # (assembly uses FP64 atomics: not bitwise reproducible on a GPU)
    # LM with float Jacobians reaches the FP64 reference's optimum (FP32 protocol)
    dev.set_jacobian_precision(True)
    prm = optimizer.LevenbergMarquardtParams.CeresDefaults() if case in util.CERES_CASES else optimizer.LevenbergMarquardtParams()
    lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, prm, device_problem=dev)
    lm.optimize()
    r = util.golden(case, "lm")["lm_errors"][-1]
    assert abs(lm.error() - r) <= 1e-5 * r, (lm.error(), r)


def linear(case):
    lp = util.load_linear_case(case)
    for which, lam in util.LINEAR_LAMBDA.items():
        dev = capi.LinearDeviceProblem(ctx, lp)
        util.check_linear_against_reference(dev, lp, util.golden(case, "out%d" % which), lam)
        dev.close()


def marginals(case):
    prob = util.load_case(case)
    ref = util.golden(case, "marg")["marg_cov"]
    m = optimizer.Marginals(ctx, prob)
    off = 0
    for v in range(prob.nvars):
        d = int(prob.var_dims[v])
        R = ref[off:off + d * d].reshape(d, d).T
        off += d * d
        if v % 5 == 0:
            assert np.abs(m.marginalCovariance(v) - R).max() <= 1e-7 * np.abs(R).max(), v
    for k, vs in enumerate(util.JOINT_SETS.get(case, [])):
        J = m.jointMarginalCovariance(vs).fullMatrix()
        R = util.golden(case, f"joint{k}")["joint_cov"].reshape(J.shape).T
        assert np.abs(J - R).max() <= 1e-7 * np.abs(R).max(), vs


def dogleg(case):
    prob = util.load_case(case)
    ref = util.golden(case, "dl")
    dl = optimizer.DoglegOptimizer(ctx, prob)
    errs = [dl.error()]
    for _ in range(min(3, len(ref["dl_errors"]) - 1)):
        dl.iterate()
        errs.append(dl.error())
    assert np.allclose(errs, ref["dl_errors"][:len(errs)], rtol=1e-7), (errs, ref["dl_errors"][:len(errs)])


def gn(case):
    prob = util.load_case(case)
    ref = util.golden(case, "gn")
    dev = capi.DeviceProblem(ctx, prob)
    errs = [dev.error()]
    for _ in range(2):
        st, e = dev.gn_iterate()
        assert st == 0
        errs.append(e)
    assert np.allclose(errs, ref["gn_errors"][:3], rtol=1e-7), (errs, ref["gn_errors"][:3])


def linear_mirror(_):
    gfg = LN.GaussianFactorGraph()
    gfg.add([5], [2 * np.eye(2)], np.ones(2))
    gfg.add([5, 9], [np.eye(2), -np.eye(2)], np.array([1.0, 2.0]))
    gfg.add([9], [np.eye(2)], np.zeros(2), np.array([0.5, 0.5]))
    x = gfg.optimize([5, 9], ctx)
    A = np.zeros((6, 4)); b = np.zeros(6)
    A[0:2, 0:2] = 2 * np.eye(2); b[0:2] = 1
    A[2:4, 0:2] = np.eye(2); A[2:4, 2:4] = -np.eye(2); b[2:4] = [1, 2]
    A[4:6, 2:4] = 2 * np.eye(2)
    sol = np.linalg.lstsq(A, b, rcond=None)[0]
    assert np.allclose(np.concatenate([x[5], x[9]]), sol, atol=1e-12)
    bt = gfg.eliminateMultifrontal([5, 9], ctx)
    assert len(bt) >= 1 and bt[-1][2] == -1
    g = gfg.gradientAtZero(ctx)
    assert np.allclose(np.concatenate([g[5], g[9]]), -A.T @ b, atol=1e-12)
    xt = {5: np.array([0.3, -0.2]), 9: np.array([1.5, 0.25])}
    r = A @ np.concatenate([xt[5], xt[9]]) - b
    assert abs(gfg.error(xt, ctx) - 0.5 * r @ r) <= 1e-12


def gnc_scenario(case):
    """gtsam_b200.gnc.GncOptimizer with the device backend against the reference's GncOptimizer (TLS and GM)."""
    from gtsam_b200 import gnc
    prob = util.load_case(case)
    for loss in ("tls", "gm"):
        ref = util.golden(case, "gnc_" + loss)
        prm = gnc.GncParams()
        prm.lossType = gnc.TLS if loss == "tls" else gnc.GM
        opt = gnc.GncOptimizer(ctx, prob, prm)
        res = opt.optimize()
        opt.backend.close()
        assert float(np.abs(opt.getWeights() - ref["gnc_weights"]).max()) <= 1e-4
        assert util.relmax(res, ref["final_values"]) <= 1e-5
    # b200_set_group_noise == a problem created with that noise (bitwise: same kernels, same inputs, no atomics in linearize)
    base = gnc.strip_robust(prob)
    w = np.random.default_rng(5).uniform(0.0, 1.0, base.nfactors)
    w[::7] = 0.0
    pw = gnc.weighted_problem(base, w)
    fresh, upd = capi.DeviceProblem(ctx, pw), capi.DeviceProblem(ctx, base)
    upd.linearize(); upd.solve(1e-3)
    for gi, g in enumerate(pw.groups):
        upd.set_group_noise(gi, g.noise_kind, g.noise)
    try:
        upd.solve(1e-3)
        raise AssertionError("solve on a stale linearization")
    except capi.B200Error:
        pass
    fresh.linearize(); upd.linearize()
    for gi in range(len(pw.groups)):
        assert np.array_equal(fresh.get_jacobians(gi), upd.get_jacobians(gi))
    assert fresh.solve(1e-3, True)[0] == upd.solve(1e-3, True)[0] == 0
    assert util.rel2(fresh.get_delta(), upd.get_delta()) <= 1e-10
    assert upd.L.b200_set_group_noise(upd.h, 99, P.NOISE_UNIT, 0, None) == 4
    assert upd.L.b200_set_group_noise(upd.h, 0, 77, 0, None) == 3
    assert upd.L.b200_set_group_noise(upd.h, 0, P.NOISE_DIAGONAL, 0, None) == 4
    fresh.close(); upd.close()


def edge(_):
    """tests/test_gpu_parity.py::test_cuda_edge_cases + API misuse: forests, empty groups, rank-deficient leaves, calls in
    the wrong order, calls that need Values on a linear problem."""
    for name, prob in util.edge_case_problems().items():
        dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
        assert abs(dev.error() - orc.error()) <= 1e-12 * max(1.0, orc.error())
        dev.linearize(); orc.linearize()
        for lam in (0.0, 1e-3):
            st, e0, e1, _ = dev.solve(lam)
            so, f0, f1, _ = orc.solve(lam)
            assert st == so, (name, lam, st, so)
            if st == 0:
                assert util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-8
                assert abs(e1 - f1) <= 1e-9 * max(1.0, f0)
        lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, device_problem=dev)
        olm = orc.lm(lm.params()._c)
        for _ in range(3):
            lm.iterate(); orc.lm_iterate(olm)
            assert abs(lm.error() - olm.state.error) <= 1e-8 * max(1.0, olm.state.error)
            assert lm.lambda_() == olm.state.lambda_
        del lm
        dev.close()
    # values snapshot / restore around a rejected step, the phase timers (what bench.py reads), joint-marginal argument checks
    prob = util.load_case("bal_tiny_s2")
    dev = capi.DeviceProblem(ctx, prob)
    dev.profile_enable(True)
    v0 = dev.get_values()
    dev.save_values()
    dev.linearize(); dev.solve(1e-3); dev.try_step(); dev.accept_step()
    assert not np.array_equal(dev.get_values(), v0)
    dev.restore_values()
    assert np.array_equal(dev.get_values(), v0)
    dev.synchronize()
    prof = dev.profile()
    assert prof["linearize"][1] + prof["linearize_small_groups"][1] >= 1 and prof["back_substitute"][1] == 1 and all(ms >= 0 for ms, _ in prof.values())
    dev.profile_enable(False)
    dev.linearize(); dev.solve(0.0)
    import ctypes
    scratch = np.zeros(32 * 32)
    for bad in ([3, 1], [1, 1], [0, prob.nvars], [-1, 2]):
        vs = np.array(bad, dtype=np.int64)
        rc = dev.L.b200_joint_marginal_covariance(dev.h, vs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 2,
                                                  scratch.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
        assert rc == P.INVALID_ARGUMENT, (bad, rc)
    dev.close()
    dev = capi.DeviceProblem(ctx, prob)
    for call in (lambda: dev.solve(0.0), lambda: dev.hessian_diagonal(), lambda: dev.get_jacobians(0), lambda: dev.try_step()):
        try:
            call()
            raise SystemExit("a call before b200_linearize / b200_solve was accepted")
        except capi.B200Error as e:
            assert e.code == P.INVALID_ARGUMENT
    dev.close()
    lp = util.load_linear_case("lin_arity8")
    ldev = capi.LinearDeviceProblem(ctx, lp)
    for call in (lambda: ldev.error(), lambda: ldev.linearize(), lambda: ldev.try_step(), lambda: ldev.set_jacobian_precision(True),
                 lambda: optimizer.LevenbergMarquardtOptimizer(ctx, lp, device_problem=ldev)):
        try:
            call()
            raise SystemExit("a call that needs Values was accepted on a linear problem")
        except capi.B200Error as e:
            assert e.code == P.INVALID_ARGUMENT
    ldev.close()


def bigfront(_):
    """Fronts of 128 columns and more through both builds of the tile dataflow (front_df_kernel<2> / <3>, emulated DMMA
    fragment layout), against the oracle."""
    from gtsam_b200 import datasets
    for minb in (2, 3):
        os.environ["B200_DF_MINB"] = str(minb)
        prob = datasets.make("sphere_tiny", layers=10, per_ring=16)
        dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
        info = dev.symbolic_info()
        assert info.max_frontal_dim + info.max_separator_dim >= 128
        dev.linearize(); orc.linearize()
        for lam in (0.0, 1e-3):
            st, e0, e1, _ = dev.solve(lam)
            so, f0, f1, _ = orc.solve(lam)
            assert st == so == 0 and util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-8 and abs(e1 - f1) <= 1e-9 * f0
        a, b = dev.conditional(info.ncliques - 1), orc.conditional(info.ncliques - 1)
        assert np.abs(a - b).max() <= 1e-7 * max(1.0, np.abs(b).max())
        dev.close()
    os.environ.pop("B200_DF_MINB", None)


def midsize(model):
    """A BAL problem large enough for long runs of points with the same cameras (several staged batches per CTA in
    leaf_point_schur_kernel, both buffers of the software pipeline in use), FP64 and FP32 storage, against the oracle in
    the same mode; then two LM iterations."""
    from gtsam_b200 import datasets
    model, _, obs = model.partition("@")     # e.g. bundler@8: 8 observations per point -> 3 tiles per thread in the Schur kernel
    prob = datasets.make("bal_tiny", ncams=30, npoints=1500 if not obs else 400, visibility="banded", camera_model=model,   # (30 cameras: the band (start + 3k) mod n holds distinct cameras)
                         obs_per_point=int(obs or 6))
    # mma = 1: the per-run Schur complement on the FP64 tensor path (leaf_point_schur_mma_kernel, 16-point batches: runs of 40
    # points = two full batches + a short one); mma = 0: the FMA-tile kernel with 4- / 6-point batches
    for f32, pb, mma in ((False, 4, 1), (True, 4, 1), (False, 4, 0), (True, 4, 0), (False, 6, 0), (True, 6, 0)):
        # (run length is sized from the SM count; at this size it would be 1, so it is forced)
        os.environ["B200_LEAF_RUN_MAX"] = "40" if mma else "24"; os.environ["B200_SCHUR_PB"] = str(pb)
        dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
        os.environ.pop("B200_LEAF_RUN_MAX"); os.environ.pop("B200_SCHUR_PB")
        dev.set_tuning("schur_mma", mma)
        if not mma:     # the other variants ride along: conditionals stored directly, 128-register linearize build
            dev.set_tuning("factor_staged", 0); dev.set_tuning("lin_variant", 4)
        dev.set_jacobian_precision(f32); orc.set_jacobian_precision(f32)
        dev.linearize(); orc.linearize()
        for lam, diag in ((1e-3, False), (1e-2, True)):
            st, e0, e1, _ = dev.solve(lam, diag)
            so, f0, f1, _ = orc.solve(lam, diag)
            assert st == so == 0 and util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-6, (f32, lam)   # additive 1e-3 damping: cond ~1e8
            assert abs(e1 - f1) <= 1e-6 * f0
        lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, optimizer.LevenbergMarquardtParams.CeresDefaults(), device_problem=dev)
        olm = orc.lm(lm.params()._c)
        for _ in range(2):
            lm.iterate(); orc.lm_iterate(olm)
            assert abs(lm.error() - olm.state.error) <= 1e-6 * olm.state.error
        del lm
        dev.close()


def leafshapes(model):
    """A mixed-shape BAL build of tests/test_point_leaf_shapes.py (fast-path points at every m, runs of 1 to 17 points,
    the generic leaves next to them), cal3_s2 up to 8 observations per point (<6, 7>) or bundler up to 4 (<9, 5>), FP64 and
    FP32 storage: the factorisation and back-substitution against that file's extended-precision backward-error checks."""
    import test_point_leaf_shapes as T
    m_max = 8 if model == "cal3_s2" else 4
    prob = T.mixed_bal(model, m_max, counts=T.SMALL_COUNTS)
    for f32 in (False, True):
        os.environ["B200_LEAF_RUN_MAX"] = "17"
        try:
            dev = capi.DeviceProblem(ctx, prob)
        finally:
            os.environ.pop("B200_LEAF_RUN_MAX")
        dev.set_jacobian_precision(f32)
        dev.linearize()
        for lam, diag in ((1e-2, False), (1e-3, True)):
            st, e0, e1, _ = dev.solve(lam, diag)
            assert st == 0
            rd = T.readout(dev, prob)
            r = T.check(prob, rd, lam, diag)
            assert max(r.values()) <= 1.0, (model, f32, lam, r)
            assert abs(e1 - T.linear_error(prob, rd)) <= 1e-9 * e0
        dev.close()


def frontshapes(_):
    """The reduced build of tests/test_front_shapes.py (fronts of at most 65 pivots, small leaves under every dataflow front,
    a chain of three dataflow fronts) through both builds of the tile dataflow (front_df_kernel<2> / <3>), amalgamation on
    and off, at every damping: elim_small_kernel, front_df_kernel, backsub_small_kernel and backsub_large_kernel against
    that file's extended-precision backward-error checks.  The emulator runs a block's threads one at a time between
    barriers and every CTA in turn, so it checks indexing and arithmetic only: it cannot see a missing fence, a flag
    published before its data, or any other memory-ordering bug."""
    import test_front_shapes as T
    lp = T.front_tree("reduced")
    for minb in (2, 3):
        for amalgamate in (True, False):
            with T.env(B200_DF_MINB=str(minb), B200_NO_AMALGAMATE=None if amalgamate else "1"):
                dev = capi.LinearDeviceProblem(ctx, lp)
            sn = dev.supernodes()
            large = T.backsub_large(T.supernode_table(sn, lp.var_dims))
            for lam, diag in T.DAMPING:
                st, e0, e1, _ = dev.solve(lam, diag)
                assert st == 0
                rd = T.readout(dev, lp)
                r, _ = T.check(lp, rd, lam, diag, sn, large)
                assert max(r.values()) <= 1.0, (minb, amalgamate, lam, diag, r)
                assert abs(e1 - T.linear_error(lp, rd)) <= 1e-9 * e0
            dev.close()


def marginalshapes(_):
    """The reduced build of tests/test_marginal_shapes.py without amalgamation (a front of 257 pivots with a separator of
    257 under a 260-pivot root, a chain of three fronts, a second root) through marginal_path_kernel and
    marginal_joint_kernel: a sample of single-variable marginals (the first and last pivots of both wide fronts, pivot
    256 of the 257-pivot front, the chain's leaf, the second root) and the joint sets of that file, against its
    extended-precision forward-error bound; joint diagonal blocks equal to the single marginals bit for bit, cross-tree
    blocks exactly zero.  Indexing and arithmetic only (see frontshapes)."""
    import test_front_shapes as FS
    import test_marginal_shapes as T
    lp = T.mbuild("reduced")
    V = T.var_of_node("reduced")
    with FS.env(B200_NO_AMALGAMATE="1"):
        dev = capi.LinearDeviceProblem(ctx, lp)
    qv = [V["A", 0], V["A", 28], V["R", 0], V["R", 27], V["R", 30], V["k0", 0], V["Q", 2]]
    singles = {v: dev.marginal_covariance(v) for v in qv}
    rd = FS.readout(dev, lp)
    sets = T.joint_sets("reduced")
    joints = [(vs, dev.joint_marginal_covariance(vs)) for vs in sets]
    sn = dev.supernodes()
    t = FS.supernode_table(sn, lp.var_dims)
    assert {257} <= set(t["f"].tolist()) and 257 in set(t["s"].tolist())
    r, _ = FS.check(lp, rd, 0.0, False, sn, FS.backsub_large(t))
    assert max(r.values()) <= 1.0, r
    rs, rj = T.check_marginals(lp, rd, singles, joints)
    assert rs <= 1.0 and rj <= 1.0, (rs, rj)
    dof = lp.dof_offsets()
    for vs, S in joints:
        o = np.concatenate([[0], np.cumsum(lp.var_dims[list(vs)])])
        for a, u in enumerate(vs):
            if u in singles:
                assert np.array_equal(S[o[a]:o[a + 1], o[a]:o[a + 1]], singles[u]), (vs, u)
        if V["Q", 0] in vs or V["Q", 1] in vs:
            q = [a for a, u in enumerate(vs) if u in (V["Q", 0], V["Q", 1])][0]
            rest = np.concatenate([np.arange(o[a], o[a + 1]) for a in range(len(vs)) if a != q])
            assert np.all(S[np.ix_(rest, np.arange(o[q], o[q + 1]))] == 0.0), vs
    dev.close()


def coverage(_):
    """Kernel instantiations no fixture reaches (tests/emu/kernel_coverage.py): PriorFactor<Point3> outside the fused
    leaves (points ordered LAST, so their cliques are interior), Dogleg with FP32 Jacobian storage on every factor family
    (gradient_kernel<T, float>)."""
    from gtsam_b200 import datasets
    b = datasets.make("bal_tiny", ncams=8, npoints=40, visibility="scattered")
    pts = np.where(b.var_type == P.VAR_POINT3)[0][:10]
    off = b.val_offsets()
    meas = np.stack([b.values[off[v]:off[v] + 3] + 0.01 for v in pts])
    pri = P.FactorGroup(P.FACTOR_PRIOR_POINT3, pts[:, None], meas, P.NOISE_DIAGONAL, np.array([0.1, 0.2, 0.3]))
    cams_first = np.concatenate([np.where(b.var_type != P.VAR_POINT3)[0], np.where(b.var_type == P.VAR_POINT3)[0]])
    pp = P.Problem(b.var_type, b.values, cams_first, list(b.groups) + [pri], cal=b.cal)
    cases = [pp, util.load_case("sphere_tiny"), util.load_case("bal_tiny_s2"), util.load_case("bal_tiny_bundler"), util.load_case("pose2_ring")]
    for prob in cases:
        for f32 in (False, True):
            dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
            dev.set_jacobian_precision(f32); orc.set_jacobian_precision(f32)
            dev.linearize(); orc.linearize()
            assert util.relmax(dev.hessian_diagonal(), orc.hessian_diagonal()) <= 1e-12
            st, e0, e1, _ = dev.solve(1e-2, True)
            so, f0, f1, _ = orc.solve(1e-2, True)
            assert st == so == 0 and util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-8
            assert abs(e0 - f0) <= 1e-11 * f0 and abs(e1 - f1) <= 1e-9 * f0
            dl = optimizer.DoglegOptimizer(ctx, prob, device_problem=dev)
            err, rad = orc.error(), 1.0
            for _ in range(3):
                dl.iterate()
                so, err, rad = orc.dogleg_iterate(err, rad)
                assert so == 0 and abs(dl.error() - err) <= 1e-7 * err and abs(dl.getDelta() - rad) <= 1e-9 * rad, (prob.name, f32, dl.error(), err, dl.getDelta(), rad)
            del dl
            dev.close()
    # Rot3::Logmap next to pi (gtsam/geometry/SO3.cpp:264-319, one branch per dominant axis) in Between / Prior residuals and
    # their Jacobians; points behind the camera (CheiralityException: zero Jacobians, residual 2 fx) for both camera models
    eye = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])
    for axis in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0.6, 0.62], [0.7, 0.1, 0.7]):
        w = np.asarray(axis, dtype=float)
        w = w / np.linalg.norm(w) * (np.pi - 2e-4)
        R, t = datasets.se3_exp(np.concatenate([w, [0.3, -0.2, 0.1]])[None, :])
        meas = datasets.pack_pose(R, t)
        btw = P.FactorGroup(P.FACTOR_BETWEEN_POSE3, np.array([[0, 1]]), meas, P.NOISE_DIAGONAL, np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6]))
        pri = P.FactorGroup(P.FACTOR_PRIOR_POSE3, np.array([[0]]), meas, P.NOISE_ISOTROPIC, np.array([0.5]))
        prob = P.Problem(np.array([P.VAR_POSE3, P.VAR_POSE3]), np.concatenate([eye, eye + 1e-3 * np.arange(12)]), np.array([0, 1]), [btw, pri])
        dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
        assert abs(dev.error() - orc.error()) <= 1e-12 * orc.error()
        dev.linearize(); orc.linearize()
        for gi in range(2):
            assert util.relmax(dev.get_jacobians(gi), orc.get_jacobians(gi)) <= 1e-9, (axis, gi)
        dev.close()
    K = np.array([[500.0, 500.0, 0.0, 320.0, 240.0]])
    behind = np.concatenate([eye, [0.1, 0.2, -3.0]])
    prob = P.Problem(np.array([P.VAR_POSE3, P.VAR_POINT3]), behind, np.array([1, 0]),
                     [P.FactorGroup(P.FACTOR_PROJECTION_CAL3S2, np.array([[0, 1]]), np.array([[1.0, 2.0]]), P.NOISE_UNIT)], K)
    cam = np.concatenate([eye, [500.0, 0.01, 0.001, 0.0, 0.0]])
    prob_b = P.Problem(np.array([P.VAR_CAM_BUNDLER, P.VAR_POINT3]), np.concatenate([cam, [0.1, 0.2, -3.0]]), np.array([1, 0]),
                       [P.FactorGroup(P.FACTOR_SFM_BUNDLER, np.array([[0, 1]]), np.array([[1.0, 2.0]]), P.NOISE_UNIT)])
    for pr in (prob, prob_b):
        dev, orc = capi.DeviceProblem(ctx, pr), O.OracleProblem(pr)
        # GenericProjectionFactor: residual 2 fx per row (ProjectionFactor.h:156-165); GeneralSFMFactor: zero residual (GeneralSFMFactor.h:132-141)
        assert dev.error() == orc.error() == (1e6 if pr is prob else 0.0)
        dev.linearize(); orc.linearize()
        J = dev.get_jacobians(0)
        assert np.all(J[:, :, :-1] == 0) and np.array_equal(J, orc.get_jacobians(0))
        dev.close()
    # Dogleg with an oversized trust region: rejected and shrunk steps (the rho < 0.25 and rho < 0 branches)
    shrunk = 0
    for name in ("sphere_tiny", "bal_tiny_s2", "pose3example"):
        prob = util.load_case(name)
        prm = optimizer.DoglegParams()
        prm.deltaInitial = 1e4
        dev, orc = capi.DeviceProblem(ctx, prob), O.OracleProblem(prob)
        dl = optimizer.DoglegOptimizer(ctx, prob, prm, device_problem=dev)
        err, rad = orc.error(), 1e4
        for _ in range(6):
            dl.iterate()
            prev = err
            so, err, rad2 = orc.dogleg_iterate(err, rad)
            if abs(prev - err) <= 1e-9 * err:
                break       # converged: the sign of rho is round-off from here on (in the reference too)
            shrunk += rad2 < rad
            rad = rad2
            assert so == 0 and abs(dl.error() - err) <= 1e-7 * err and abs(dl.getDelta() - rad) <= 1e-9 * rad, (name, dl.error(), err, dl.getDelta(), rad)
        del dl
        dev.close()
    assert shrunk >= 1
    # the device order of the projection groups (leaf-visit order, create_problem) is internal: Jacobians come back in the caller's
    # order and every result is the same as with graph-order storage (B200_NO_FACTOR_REORDER=1)
    for name in ("bal_tiny_s2", "bal_tiny_bundler", "bal_small_metis"):
        prob = util.load_case(name)
        res = []
        for off in (False, True):
            if off:
                os.environ["B200_NO_FACTOR_REORDER"] = "1"
            try:
                dev = capi.DeviceProblem(ctx, prob)
            finally:
                os.environ.pop("B200_NO_FACTOR_REORDER", None)
            dev.linearize()
            st, e0, e1, _ = dev.solve(1e-2, True)
            res.append(([dev.get_jacobians(gi) for gi in range(len(prob.groups))], dev.get_delta(), e0, e1, dev.hessian_diagonal()))
            dev.close()
        for Ja, Jb in zip(res[0][0], res[1][0]):
            assert np.array_equal(Ja, Jb), name
        assert util.rel2(res[0][1], res[1][1]) <= 1e-9 and abs(res[0][2] - res[1][2]) <= 1e-12 * res[1][2] and abs(res[0][3] - res[1][3]) <= 1e-9 * res[1][2]
        assert util.relmax(res[0][4], res[1][4]) <= 1e-12
    # ticket order of the dataflow tiles across levels (B200_DF_ORDER=1, with and without lagged trailing columns): the emulator runs
    # the CTAs in ticket order, one after the other, so a dependency that pointed forwards would time out instead of passing
    for lag in ("0", "2", "5"):
        os.environ["B200_DF_ORDER"] = "1"; os.environ["B200_DF_LAG"] = lag
        try:
            for name in ("sphere_small_colamd", "sphere_small_metis", "bal_small_metis"):
                prob = util.load_case(name)
                dev = capi.DeviceProblem(ctx, prob)
                util.check_against_dump(dev, prob, util.golden(name, "dump1"), 1e-2, 1)
                dev.close()
        finally:
            os.environ.pop("B200_DF_ORDER"); os.environ.pop("B200_DF_LAG")


def allocfail(_):
    """Each allocation a call makes fails in turn (tests/emu/cuda_fake_runtime.cpp): the call returns B200_CUDA_ERROR and
    leaves as many blocks allocated as there were before it; b200_set_jacobian_precision leaves the problem as it was."""
    import ctypes as C
    from gtsam_b200 import datasets
    L = ctx.L
    L.b200_emu_live_allocs.restype = C.c_long
    L.b200_emu_fail_alloc_in.argtypes = [C.c_long]

    def each_failure(what, call, after=None):
        k = 0
        while True:
            k += 1
            live = L.b200_emu_live_allocs()
            L.b200_emu_fail_alloc_in(k)
            rc = call()
            L.b200_emu_fail_alloc_in(0)
            if rc == P.OK:
                break
            assert rc == P.CUDA_ERROR, (what, k, rc)
            assert L.b200_emu_live_allocs() == live, (what, "allocation %d failed" % k, L.b200_emu_live_allocs() - live, "blocks leaked")
            if after:
                after()
        assert k > 1, (what, "no allocation")

    def create(what, fn, desc):
        def call():
            h = C.c_void_p()
            live = L.b200_emu_live_allocs()
            rc = fn(ctx.h, C.byref(desc), C.byref(h))
            if rc == P.OK:
                L.b200_problem_destroy(h)
                assert L.b200_emu_live_allocs() == live, (what, "b200_problem_destroy")
            return rc
        each_failure(what, call)

    for name, prob in (("bal_small_metis", util.load_case("bal_small_metis")), ("bigfront", datasets.make("sphere_tiny", layers=10, per_ring=16))):
        desc, keep = prob.c_desc()
        create(name, L.b200_problem_create, desc)
    lp = util.load_linear_case("lin_random_nary")
    desc, keep = lp.c_desc()
    create("lin_random_nary", L.b200_linear_create, desc)
    prob = util.load_case("bal_tiny_s2")
    dev = capi.DeviceProblem(ctx, prob)

    def dl_create():
        h = C.c_void_p()
        rc = L.b200_dl_create(dev.h, 1.0, C.byref(h))
        if rc == P.OK:
            L.b200_dl_destroy(h)
        return rc
    each_failure("b200_dl_create", dl_create)
    vs, cov = np.array([0, 1], dtype=np.int64), np.zeros(128 * 128)
    joint = lambda: L.b200_joint_marginal_covariance(dev.h, vs.ctypes.data_as(C.POINTER(C.c_int64)), 2, cov.ctypes.data_as(C.POINTER(C.c_double)))  # noqa: E731
    assert joint() == P.OK     # (the marginals' own buffers, kept by the problem, exist from here on)
    each_failure("b200_joint_marginal_covariance", joint)

    def unchanged():
        assert L.b200_get_jacobian_precision(dev.h) == 0
        dev.restore_values()      # (the dump check accepts a step)
        util.check_against_dump(dev, prob, util.golden("bal_tiny_s2", "dump1"), 1e-2, 1)
    dev.save_values()
    each_failure("b200_set_jacobian_precision", lambda: L.b200_set_jacobian_precision(dev.h, 1), unchanged)
    assert L.b200_get_jacobian_precision(dev.h) == 1
    dev.close()


SCEN = dict(allocfail=allocfail, coverage=coverage, leafshapes=leafshapes, frontshapes=frontshapes, marginalshapes=marginalshapes, midsize=midsize, edge=edge, bigfront=bigfront, gnc=gnc_scenario, typed=typed, fp32=fp32, linear=linear, marginals=marginals, dogleg=dogleg, gn=gn, mirror=linear_mirror)
for arg in sys.argv[2:]:
    kind, case = arg.split(":")
    t = time.time()
    SCEN[kind](case)
    print("EMU_OK %s %.1fs" % (arg, time.time() - t), flush=True)
print("EMU_LAUNCHES", ctx.launch_count())
