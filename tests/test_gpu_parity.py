"""GPU: the CUDA path, called through the C-ABI, against (1) the golden vectors
of the unmodified reference, (2) the C oracle on seeded mid-size problems and
(3) size-independent properties at BASELINE.json's full sizes.

Tolerances (FP64 path, SURVEY.md §8c): whitened [A|b] max-abs-diff <= 1e-12
relative; graph.error rel <= 1e-12; delta rel-2-norm <= 1e-8 (conditioning
limited, FP64 atomics make Hessian sums order dependent); LM traces: same
accept/reject + lambda sequence, errors rel <= 1e-7."""
import numpy as np
import pytest

import util
from gtsam_b200 import capi, datasets, optimizer, problem as P
from oracle import oracle_py as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", util.CASES)
@pytest.mark.parametrize("kind,lam,diag", [("dump0", 0.0, 0), ("dump1", 1e-2, 1)])
def test_cuda_matches_reference_dump(gpu_ctx, case, kind, lam, diag):
    prob = util.load_case(case)
    dev = capi.DeviceProblem(gpu_ctx, prob)
    util.check_against_dump(dev, prob, util.golden(case, kind), lam, diag)
    dev.close()


@pytest.mark.parametrize("case", util.CASES)
def test_cuda_lm_trace_matches_reference(gpu_ctx, case):
    prob = util.load_case(case)
    ref = util.golden(case, "lm")
    prm = optimizer.LevenbergMarquardtParams.CeresDefaults() if case in util.CERES_CASES else optimizer.LevenbergMarquardtParams()
    prm.maxIterations = 100 if case.startswith("dub") else 30
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, prob, prm)
    errs, lams, inner = [], [], []
    prm.iterationHook = lambda it, old, new: (errs.append(new), lams.append(lm.lambda_()), inner.append(lm.getInnerIterations()))
    e0 = lm.error()
    lm.optimize()
    errs, lams, inner = [e0] + errs, [prm.lambdaInitial] + lams, [0] + inner
    assert len(errs) == len(ref["lm_errors"])
    assert np.allclose(errs, ref["lm_errors"], rtol=1e-5 if case.startswith("dub") else 1e-7, atol=1e-10)
    assert np.allclose(lams, ref["lm_lambdas"], rtol=1e-12)
    assert inner == list(ref["lm_inner"])
    assert util.relmax(lm.values(), ref["final_values"]) <= (1e-3 if case.startswith("dub") else 1e-6)


def test_cuda_reference_end_to_end_golden(gpu_ctx):
    """tests/testGeneralSFMFactorB.cpp:44-63 through the drop-in: 0.0199833 +- 1e-5."""
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, util.load_case("dubrovnik_3_7_unit"))
    lm.optimize()
    assert abs(lm.error() - 0.0199833) < 1e-5


@pytest.mark.parametrize("case", ["bal_tiny_s2", "sphere_tiny", "sphere_small_colamd", "sphere_tiny_gaussian"])
def test_cuda_dogleg_trace(gpu_ctx, case):
    """DoglegOptimizer trace (errors + trust-region radii) against the reference's, deltaInitial = 1."""
    prob = util.load_case(case)
    ref = util.golden(case, "dl")
    dl = optimizer.DoglegOptimizer(gpu_ctx, prob)
    errs, deltas = [dl.error()], [dl.getDelta()]
    for _ in range(len(ref["dl_errors"]) - 1):
        dl.iterate()
        errs.append(dl.error())
        deltas.append(dl.getDelta())
    assert np.allclose(errs, ref["dl_errors"], rtol=1e-8)
    assert np.allclose(deltas, ref["dl_deltas"], rtol=1e-7)
    assert util.relmax(dl.values(), ref["final_values"]) <= 1e-6


def test_pinned_host_buffers_copy_directly(gpu_ctx):
    """b200_set_values / b200_get_values with page-locked caller buffers (direct DMA) == pageable path."""
    import torch
    prob = util.load_case("bal_tiny_s2")
    dp = capi.DeviceProblem(gpu_ctx, prob)
    e0 = dp.error()
    pinned = torch.from_numpy(prob.values.copy()).pin_memory().numpy()
    pinned += 1e-3
    dp.set_values(pinned)
    e1 = dp.error()
    dp.set_values(np.array(pinned))            # pageable copy of the same numbers
    assert dp.error() == e1 and e1 != e0
    out = torch.empty(pinned.size, dtype=torch.float64).pin_memory().numpy()
    assert dp.get_values(out) is out
    assert np.array_equal(out, pinned) and np.array_equal(dp.get_values(), pinned)
    dp.close()


def test_cuda_dogleg_optimize_mid_size(gpu_ctx):
    """Dogleg on a mid-size BAL problem converges to the LM optimum (size-independent property)."""
    from gtsam_b200 import datasets
    prob = datasets.bal(ncams=23, npoints=4000, seed=2)
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, prob)
    lm.optimize()
    dl = optimizer.DoglegOptimizer(gpu_ctx, prob)
    e0 = dl.error()
    dl.optimize()
    assert dl.error() < e0 and abs(dl.error() - lm.error()) <= 1e-3 * max(1.0, lm.error())


@pytest.mark.parametrize("case", ["sphere_tiny", "sphere_small_colamd"])
def test_cuda_gn_trace(gpu_ctx, case):
    prob = util.load_case(case)
    ref = util.golden(case, "gn")
    gn = optimizer.GaussNewtonOptimizer(gpu_ctx, prob)
    errs = [gn.error()]
    for _ in range(len(ref["gn_errors"]) - 1):
        gn.iterate()
        errs.append(gn.error())
    assert np.allclose(errs, ref["gn_errors"], rtol=1e-8)


MID = [("bal_tiny", dict(ncams=23, npoints=3000, visibility="scattered")),
       ("bal_tiny", dict(ncams=40, npoints=4000, visibility="banded", camera_model="bundler")),
       ("sphere_tiny", dict(layers=14, per_ring=24)),                       # large fronts (natural ordering)
       ("sphere_tiny", dict(layers=14, per_ring=24, ordering="reverse"))]


@pytest.mark.parametrize("name,kw", MID)
@pytest.mark.parametrize("lam,diag", [(0.0, False), (1e-3, False), (1e-2, True)])
def test_cuda_matches_oracle_mid_size(gpu_ctx, name, kw, lam, diag):
    prob = datasets.make(name, **kw)
    dev, orc = capi.DeviceProblem(gpu_ctx, prob), O.OracleProblem(prob)
    eo = orc.error()
    assert abs(dev.error() - eo) <= 1e-12 * eo
    dev.linearize(); orc.linearize()
    for gi in range(len(prob.groups)):
        assert util.relmax(dev.get_jacobians(gi), orc.get_jacobians(gi)) <= 1e-12
    assert util.relmax(dev.hessian_diagonal(), orc.hessian_diagonal()) <= 1e-12
    st, e0, e1, _ = dev.solve(lam, diag)
    so, f0, f1, _ = orc.solve(lam, diag)
    assert st == so == 0
    # undamped BAL systems are conditioning-limited (two sigma=0.1 priors pin the gauge)
    assert util.rel2(dev.get_delta(), orc.get_delta()) <= (1e-8 if lam > 0 else 1e-6)
    assert abs(e0 - f0) <= 1e-12 * f0 and abs(e1 - f1) <= 1e-9 * f0
    ne, no = dev.try_step(), orc.try_step()
    assert abs(ne - no) <= 1e-8 * max(1.0, no)
    dev.accept_step(); orc.accept_step()
    assert util.relmax(dev.get_values(), orc.get_values()) <= 1e-9
    # conditionals of a few cliques, incl. the root
    info = dev.symbolic_info()
    for c in sorted({0, info.ncliques // 2, info.ncliques - 1}):
        a, b = dev.conditional(c), orc.conditional(c)
        assert np.abs(a - b).max() <= 1e-7 * max(1.0, np.abs(b).max())
    dev.close()


def test_cuda_indeterminate_system_reported(gpu_ctx):
    """Gauge-free BAL (no priors): the undamped system is singular -> B200_INDETERMINATE
    with a nearby variable, like IndeterminantLinearSystemException; LM recovers by raising lambda."""
    prob = datasets.make("bal_tiny")
    prob.groups = prob.groups[:1]
    prob = P.Problem(prob.var_type, prob.values, prob.ordering, prob.groups, prob.cal)
    dev, orc = capi.DeviceProblem(gpu_ctx, prob), O.OracleProblem(prob)
    dev.linearize(); orc.linearize()
    st, _, _, fv = dev.solve(0.0)
    so, _, _, fo = orc.solve(0.0)
    assert so == P.INDETERMINATE and st == P.INDETERMINATE and fv >= 0
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, prob, device_problem=dev)
    e0 = lm.error()
    lm.iterate()
    assert lm.error() < e0


def test_cuda_cheirality(gpu_ctx):
    pose = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])
    K = np.array([[500.0, 500.0, 0.0, 320.0, 240.0]])
    prob = P.Problem(np.array([P.VAR_POSE3, P.VAR_POINT3]), np.concatenate([pose, [0.1, 0.2, -3.0]]), np.array([1, 0]),
                     [P.FactorGroup(P.FACTOR_PROJECTION_CAL3S2, np.array([[0, 1]]), np.array([[1.0, 2.0]]), P.NOISE_UNIT)], K)
    dev = capi.DeviceProblem(gpu_ctx, prob)
    dev.linearize()
    J = dev.get_jacobians(0)[0]
    assert np.all(J[:, :9] == 0) and np.allclose(J[:, 9], -1000.0)
    assert abs(dev.error() - 1e6) < 1e-6


def test_cuda_logmap_near_pi_and_bundler_cheirality(gpu_ctx):
    """Branches no fixture reaches (found with gcov on the host-emulation build, where they pass): Rot3::Logmap next to pi
    (gtsam/geometry/SO3.cpp:264-319, one branch per dominant axis) inside Between / Prior residuals and Jacobians, and
    GeneralSFMFactor's CheiralityException handling (GeneralSFMFactor.h:132-141: zero residual, zero Jacobians) — device
    vs the oracle (pinned on the reference's near-pi known answers, tests/test_oracle_golden.py)."""
    from gtsam_b200 import datasets
    from oracle import oracle_py as O
    eye = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])
    worst = 0.0
    for axis in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [0.5, 0.6, 0.62], [0.7, 0.1, 0.7]):
        w = np.asarray(axis, dtype=float)
        w = w / np.linalg.norm(w) * (np.pi - 2e-4)
        R, t = datasets.se3_exp(np.concatenate([w, [0.3, -0.2, 0.1]])[None, :])
        meas = datasets.pack_pose(R, t)
        btw = P.FactorGroup(P.FACTOR_BETWEEN_POSE3, np.array([[0, 1]]), meas, P.NOISE_DIAGONAL, np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6]))
        pri = P.FactorGroup(P.FACTOR_PRIOR_POSE3, np.array([[0]]), meas, P.NOISE_ISOTROPIC, np.array([0.5]))
        prob = P.Problem(np.array([P.VAR_POSE3, P.VAR_POSE3]), np.concatenate([eye, eye + 1e-3 * np.arange(12)]), np.array([0, 1]), [btw, pri])
        dev, orc = capi.DeviceProblem(gpu_ctx, prob), O.OracleProblem(prob)
        worst = max(worst, abs(dev.error() - orc.error()) / orc.error() * 1e3)      # 1e-12 on the error ~ 1e-9 on the scale below
        dev.linearize(); orc.linearize()
        for gi in range(2):
            worst = max(worst, util.relmax(dev.get_jacobians(gi), orc.get_jacobians(gi)))
        dev.close()
    cam = np.concatenate([eye, [500.0, 0.01, 0.001, 0.0, 0.0]])
    prob_b = P.Problem(np.array([P.VAR_CAM_BUNDLER, P.VAR_POINT3]), np.concatenate([cam, [0.1, 0.2, -3.0]]), np.array([1, 0]),
                       [P.FactorGroup(P.FACTOR_SFM_BUNDLER, np.array([[0, 1]]), np.array([[1.0, 2.0]]), P.NOISE_UNIT)])
    dev = capi.DeviceProblem(gpu_ctx, prob_b)
    dev.linearize()
    zero = dev.error() == 0.0 and bool(np.all(dev.get_jacobians(0) == 0))
    dev.close()
    if not (worst <= 1e-9 and zero):
        pytest.fail(f"near-pi Logmap / Bundler cheirality: off: worst {worst:.3g}, cheirality zero {zero}")


def _normal_equation_residual(prob, dev, lam):
    """|J^T (J d - b) + lam d| / |J^T b| from the device Jacobians, with scipy.sparse."""
    import scipy.sparse as sp
    dof = prob.dof_offsets()
    n = int(dof[-1])
    rows, cols, vals, bs = [], [], [], []
    r0 = 0
    for gi, g in enumerate(prob.groups):
        J = dev.get_jacobians(gi)
        d = P.FACTOR_DIM[g.type]
        rr = r0 + (np.arange(g.count)[:, None] * d + np.arange(d)[None]).astype(np.int64)     # (count, d)
        c0 = 0
        for a, vt in enumerate(P.FACTOR_VAR_TYPES[g.type]):
            nv = P.VAR_DIM[vt]
            cc = dof[g.keys[:, a]][:, None] + np.arange(nv)[None]                                # (count, nv)
            rows.append(np.repeat(rr[:, :, None], nv, 2).ravel())
            cols.append(np.repeat(cc[:, None, :], d, 1).ravel())
            vals.append(J[:, :, c0:c0 + nv].ravel())
            c0 += nv
        bs.append(J[:, :, -1].ravel())
        r0 += g.count * d
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(r0, n))
    b = np.concatenate(bs)
    dl = dev.get_delta()
    g0 = A.T @ b
    return float(np.linalg.norm(A.T @ (A @ dl - b) + lam * dl) / np.linalg.norm(g0)), A, b, dl


@pytest.mark.parametrize("workload,lam", [("bal_c3", 1e-5), ("sphere2500", 0.0), ("bal_1m", 1e-5)])
def test_full_size_normal_equations(gpu_ctx, workload, lam):
    """BASELINE.json configs[2] / configs[1] at full size: delta satisfies the damped normal
    equations to 1e-9 and the reported linear errors equal 0.5|b|^2 and 0.5|A delta - b|^2."""
    prob = datasets.make(workload)
    dev = capi.DeviceProblem(gpu_ctx, prob)
    dev.linearize()
    st, e0, e1, _ = dev.solve(lam)
    assert st == 0
    res, A, b, dl = _normal_equation_residual(prob, dev, lam)
    assert res <= 1e-9, res
    assert abs(e0 - 0.5 * b @ b) <= 1e-11 * e0
    r = A @ dl - b
    assert abs(e1 - 0.5 * r @ r) <= 1e-9 * e0
    ne = dev.try_step()
    if lam > 0:   # a damped step must decrease the error; a raw GN step on a noisy sphere need not
        assert ne < dev.error()
    dev.close()


def test_full_size_lm_iteration_decreases_error(gpu_ctx):
    prob = datasets.make("bal_c3")
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, prob)
    e0 = lm.error()
    lm.iterate()
    assert lm.error() < 0.1 * e0 and lm.iterations() == 1


@pytest.mark.parametrize("name", ["priors_only", "two_components_empty_group", "single_observation_points"])
def test_cuda_edge_cases(gpu_ctx, name):
    """Forests, empty groups, rank-deficient leaves: same status, delta and LM behaviour as the oracle."""
    prob = util.edge_case_problems()[name]
    dev, orc = capi.DeviceProblem(gpu_ctx, prob), O.OracleProblem(prob)
    assert abs(dev.error() - orc.error()) <= 1e-12 * max(1.0, orc.error())
    dev.linearize(); orc.linearize()
    for lam in (0.0, 1e-3):
        st, e0, e1, _ = dev.solve(lam)
        so, f0, f1, _ = orc.solve(lam)
        assert st == so
        if st == 0:
            assert util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-8
            assert abs(e1 - f1) <= 1e-9 * max(1.0, f0)
    lm = optimizer.LevenbergMarquardtOptimizer(gpu_ctx, prob, device_problem=dev)
    olm = orc.lm(lm.params()._c)
    for _ in range(3):
        lm.iterate(); orc.lm_iterate(olm)
        assert abs(lm.error() - olm.state.error) <= 1e-8 * max(1.0, olm.state.error)
        assert lm.lambda_() == olm.state.lambda_


def test_tile_dataflow_fronts_match_oracle(gpu_ctx):
    """front_df_kernel (the default): every non-leaf front of the tree factored as tiles of ONE launch (pieces published
    through flags, Schur complements extend-added across levels inside the launch), on graphs whose fronts span several
    128 x 32 tiles and several pivot blocks, with supernode amalgamation on: delta, linear error and the root conditional
    against the oracle, and every reference clique's conditional read back out of its supernode."""
    for kw in (dict(layers=14, per_ring=24), dict(layers=14, per_ring=24, ordering="reverse")):
        prob = datasets.make("sphere_tiny", **kw)
        dev, orc = capi.DeviceProblem(gpu_ctx, prob), O.OracleProblem(prob)
        info = dev.symbolic_info()
        assert info.supernode_max_frontal_dim + info.supernode_max_separator_dim >= 256 and info.supernodes < info.ncliques
        dev.linearize(); orc.linearize()
        for lam in (0.0, 1e-3):
            st, e0, e1, _ = dev.solve(lam)
            so, f0, f1, _ = orc.solve(lam)
            assert st == so == 0
            assert util.rel2(dev.get_delta(), orc.get_delta()) <= 1e-8
            assert abs(e1 - f1) <= 1e-9 * f0
        worst = 0.0
        for c in list(range(0, info.ncliques, max(1, info.ncliques // 40))) + [info.ncliques - 1]:
            a, b = dev.conditional(c), orc.conditional(c)
            worst = max(worst, np.abs(a - b).max() / max(1.0, np.abs(b).max()))
        assert worst <= 1e-7, worst
        dev.close()
