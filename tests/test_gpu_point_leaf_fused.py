"""The BAL point leaves on the device with long runs: leaf_point_fused_mma_kernel (schur_mma = 1, the default) against the
split path (schur_mma = 0: leaf_point_factor_kernel + the FMA-tile leaf_point_schur_kernel) and against the oracle.

The GPU fixtures elsewhere get runs of at most a few points (the run length is sized from the SM count), so no warp there
takes a second mini-batch and the kernel's double-buffered cp.async pipeline never runs on hardware.  Here runs are forced
to 64 points (16 mini-batches, 4 per warp, a short last one where a camera set has a remainder), for 6-dof cameras at 5 and
6 observations per point (5 and 6 column strips) and 9-dof cameras at 8 (10 strips), with FP64 and FP32 Jacobian storage:
  * the point conditionals [R S' d'] of an additively damped solve (lambda = 1e-2) are bitwise those of the split path (both
    go through the same per-point arithmetic; diagonal damping would bring in the Hessian diagonal, summed with atomics);
  * delta of a diagonally damped solve agrees with the split path to 1e-10 and with the oracle to 1e-8 (FP32 storage: 1e-5,
    the oracle rounds its own FP64 Jacobians to float, tests/test_gpu_precision.py);
  * the LM error after two iterations agrees with the split path to 1e-10 and with the oracle to 1e-7 (FP32 storage: both
    1e-5, the FP32 protocol of SURVEY 8(c)).
Own process; strict: any mismatch, crash or timeout fails with stderr."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import os, sys
import ctypes as C
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import util
from gtsam_b200 import capi, datasets, optimizer, problem as P
from oracle import oracle_py as O
ctx = capi.Context(0)
checked = 0
for model, obs in (("cal3_s2", 5), ("cal3_s2", 6), ("bundler", 8)):
    prob = datasets.make("bal_tiny", ncams=30, npoints=3000, visibility="banded", camera_model=model, obs_per_point=obs)
    for f32 in (False, True):
        os.environ["B200_LEAF_RUN_MAX"] = "64"
        devs = {{mma: capi.DeviceProblem(ctx, prob) for mma in (1, 0)}}
        os.environ.pop("B200_LEAF_RUN_MAX")
        orc = O.OracleProblem(prob)
        orc.set_jacobian_precision(f32)
        orc.linearize()
        so, f0, f1, _ = orc.solve(1e-2, True)
        assert so == 0
        d_orc = orc.get_delta()
        tol_d, tol_e = (1e-5, 1e-5) if f32 else (1e-8, 1e-9)
        delta, conds = {{}}, {{}}
        for mma, dev in devs.items():
            dev.set_tuning("schur_mma", mma)
            dev.set_jacobian_precision(f32)
            dev.linearize()
            assert dev.solve(1e-2, False)[0] == 0
            # the conditionals of the point cliques (one Point3 frontal)
            fp, fv, sp, sv, _ = dev.cliques()
            dims = prob.var_dims
            out = []
            for c in range(len(fp) - 1):
                if fp[c + 1] - fp[c] != 1 or prob.var_type[fv[fp[c]]] != P.VAR_POINT3:
                    continue
                s = int(dims[sv[sp[c]:sp[c + 1]]].sum())
                m = np.zeros(3 * (3 + s + 1))
                capi._check(dev.L.b200_get_conditional(dev.h, c, m.ctypes.data_as(C.POINTER(C.c_double))))
                out.append(m)
            conds[mma] = out
            st, e0, e1, _ = dev.solve(1e-2, True)
            assert st == 0 and abs(e1 - f1) <= tol_e * f0, (model, obs, f32, mma, st, e1, f1)
            delta[mma] = dev.get_delta()
            assert util.rel2(delta[mma], d_orc) <= tol_d, (model, obs, f32, mma, util.rel2(delta[mma], d_orc))
        assert len(conds[1]) == len(conds[0]) > 0
        bad = [i for i, (a, b) in enumerate(zip(conds[1], conds[0])) if not np.array_equal(a, b)]
        assert not bad, (model, obs, f32, "conditionals differ", len(bad), len(conds[1]),
                         max(float(np.abs(conds[1][i] - conds[0][i]).max()) for i in bad))
        assert util.rel2(delta[1], delta[0]) <= 1e-10, (model, obs, f32, util.rel2(delta[1], delta[0]))
        errs = {{}}
        for mma, dev in devs.items():
            lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, device_problem=dev)
            for _ in range(2):
                lm.iterate()
            errs[mma] = lm.error()
            if mma == 1:
                olm = orc.lm(lm.params()._c)
                for _ in range(2):
                    orc.lm_iterate(olm)
                assert abs(errs[1] - olm.state.error) <= (1e-5 if f32 else 1e-7) * olm.state.error, (model, obs, f32, errs[1], olm.state.error)
            del lm
            dev.close()
        # (FP32 storage: two LM iterations of the same path already differ by up to ~1e-6 from run to run: the atomics of
        # the extend-add reorder sums, and the second linearization rounds its Jacobians to float)
        assert abs(errs[1] - errs[0]) <= (1e-5 if f32 else 1e-10) * errs[0], (model, obs, f32, errs)
        checked += len(conds[1])
print("FUSED_OK", checked)
"""


def test_point_leaf_fused_matches_split_path_and_oracle():
    try:
        out = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT)], capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired:
        pytest.fail("point-leaf fused kernel: timed out")
    lines = [l for l in out.stdout.splitlines() if l.startswith("FUSED_OK")]
    if not lines:
        pytest.fail("point-leaf fused kernel: did not complete: " + out.stderr[-3000:])
    assert int(lines[-1].split()[1]) > 0
