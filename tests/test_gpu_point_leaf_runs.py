"""The BAL point leaves on the device with runs of several hundred points and uneven cuts.

The leaf runs are sized to the GPU (engine.cu): on the large workloads a run is a whole camera set of 300 to 600 points,
split evenly where the kind would not fill the GPU otherwise.  The other GPU fixtures build runs of at most 65 points.  Here
`mixed_bal` (tests/test_point_leaf_shapes.py) gets camera sets of 301, 450 and 619 points (mini-batch counts 76, 113 and 155;
last mini-batches of 1, 2 and 3 points), for 6-dof cameras (leaf_point_fused_mma_kernel<6, 5>) and 9-dof cameras (<9, 5>),
with FP64 and FP32 Jacobian storage, at the default run rule, at runs cut greedily at 200 points (200 + 101, 200 + 200 + 50,
3 x 200 + 19) and at whole camera sets (B200_LEAF_RUN_MAX = 1024).  Per cell:
  * every check of the extended-precision backward-error checker of test_point_leaf_shapes.py, and the linear error;
  * delta against the oracle (1e-8; FP32 storage: 1e-5 with the oracle in FP32 mode);
  * the point conditionals of the additively damped solve bitwise equal to the split path's (schur_mma = 0);
  * with FP64 storage, the LM error after one iteration against the oracle's (1e-7).
Own process; strict: any mismatch, crash or timeout fails with stderr."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import os, sys
import numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {root!r} + "/tests")
import util
import test_point_leaf_shapes as T
from gtsam_b200 import capi, optimizer
from oracle import oracle_py as O
ctx = capi.Context(0)
cells = 0
for model, m_max in (("cal3_s2", 6), ("bundler", 4)):
    prob = T.mixed_bal(model, m_max, m_min=m_max - 1, counts=(301, 450, 619))
    print(model, "m", m_max - 1, "-", m_max, "-> leaf_point_fused_mma_kernel<%d, %d>" % T.instantiation(model, m_max), flush=True)
    for f32 in (False, True):
        orc = O.OracleProblem(prob)
        orc.set_jacobian_precision(f32)
        orc.linearize()
        ref = {{}}
        for lam, diag in ((1e-2, False), (1e-3, True)):
            assert orc.solve(lam, diag)[0] == 0
            ref[(lam, diag)] = orc.get_delta()
        del orc
        for run in (None, 200, 1024):
            if run:
                os.environ["B200_LEAF_RUN_MAX"] = str(run)
            try:
                dev = capi.DeviceProblem(ctx, prob)
                split = capi.DeviceProblem(ctx, prob)
            finally:
                os.environ.pop("B200_LEAF_RUN_MAX", None)
            split.set_tuning("schur_mma", 0)
            for d in (dev, split):
                d.set_jacobian_precision(f32); d.linearize()
            for lam, diag in ((1e-2, False), (1e-3, True)):
                cell = "%s %s run %s lam %g %s" % (model, "fp32" if f32 else "fp64", run or "default", lam, "diag" if diag else "add")
                st, e0, e1, _ = dev.solve(lam, diag)
                assert st == 0, (cell, st)
                rd = T.readout(dev, prob)
                r = T.check(prob, rd, lam, diag)
                le = abs(e1 - T.linear_error(prob, rd)) / (1e-9 * e0)
                print(cell, " ", T.fmt(r), " e1 %.3g" % le, flush=True)
                assert max(r.values()) <= 1.0 and le <= 1.0, (cell, r, le)
                rel = util.rel2(rd["delta"], ref[(lam, diag)])
                assert rel <= (1e-5 if f32 else 1e-8), (cell, "delta vs oracle", rel)
                if not diag:
                    assert split.solve(lam, diag)[0] == 0
                    other = T.readout(split, prob)
                    pc = T.point_cliques(prob, rd)
                    bad = [c for c in pc if not np.array_equal(rd["conds"][c], other["conds"][c])]
                    assert not bad, (cell, "point conditionals differ from the split path", len(bad), len(pc))
                cells += 1
            if not f32:
                lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, device_problem=dev)
                lm.iterate()
                orc = O.OracleProblem(prob)
                olm = orc.lm(lm.params()._c)
                orc.lm_iterate(olm)
                assert abs(lm.error() - olm.state.error) <= 1e-7 * olm.state.error, (model, run, lm.error(), olm.state.error)
                del lm, orc
            dev.close()
            split.close()
print("RUNS_OK", cells)
"""


def test_point_leaf_long_runs_on_gpu():
    try:
        out = subprocess.run([sys.executable, "-c", SCRIPT.format(root=ROOT)], capture_output=True, text=True, timeout=900)
    except subprocess.TimeoutExpired:
        pytest.fail("point-leaf long runs: timed out")
    print(out.stdout)
    lines = [l for l in out.stdout.splitlines() if l.startswith("RUNS_OK")]
    if not lines:
        pytest.fail("point-leaf long runs: did not complete: " + out.stdout[-2000:] + out.stderr[-3000:])
    assert int(lines[-1].split()[1]) == 24
