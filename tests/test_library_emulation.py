"""The WHOLE library executed on the CPU: gtsam_b200/csrc/engine.cu + kernels.cuh compiled by g++ with -DB200_EMULATE
against tests/emu/cuda_emu_full.h (every CUDA thread a fiber of one host thread, __syncthreads / __syncwarp / warp shuffles as
barriers + exchanges, cp.async a plain copy) and tests/emu/cuda_fake_runtime.cpp (device memory = host
memory) — the same source the GPU build compiles, through the same C-ABI and the same Python mirror, against the same
golden vectors of the unmodified reference.

It is how the code written after this round's GPU budget was spent gets exercised end to end before its first hardware
run: the GaussianFactorGraph level (JacobianFactor / HessianFactor groups), the FP32-storage mode through the float
instantiations of the leaf kernels (cp.async staging included), the Pose2 factor family, METIS-ordered BAL, the joint
marginal kernel — next to paths that are also validated on the GPU (the BAL point-leaf kernels, the tile-dataflow fronts,
the flag-chained back-substitution, Dogleg, Gauss-Newton, LM), which makes the emulation itself credible.  It checks
logic and arithmetic, not the GPU: no memory-model subtleties, no performance.  The scenario groups run as parallel
processes (tests/emu/run_scenarios.py).

The scenario groups run against an AddressSanitizer build of the same sources when libasan is present: device memory is
the host heap there, so an out-of-bounds access of any kernel (global or shared memory) or of the host code is a test
failure — the part of compute-sanitizer's memcheck that does not need the GPU.  They also run with the threads of a
block scheduled in a freshly shuffled order between barriers (B200_EMU_ORDER, tests/emu/cuda_emu_full.h): a missing
__syncthreads / __syncwarp, or reliance on warp lock-step, changes results with the order — the emulator's stand-in for
racecheck.  All scenarios pass in ascending, reverse and shuffled order."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
LIB = os.path.join(EMU, "_build", "libgtsam_b200_emu.so")
LIB_ASAN = os.path.join(EMU, "_build", "libgtsam_b200_emu_asan.so")
CSRC = os.path.join(ROOT, "gtsam_b200", "csrc")

GROUPS = [
    # every typed golden case: both reference dumps (every stage incl. all conditionals) + the LM trace
    ["typed:bal_tiny_s2", "typed:bal_tiny_bundler", "typed:bal_tiny_colamd", "typed:bal_tiny_body_sensor", "typed:bal_tiny_tukey",
     "typed:bal_tiny_fair", "typed:bal_small_metis", "typed:pose2_ring", "typed:pose2_ring_colamd"],
    ["typed:sphere_tiny", "typed:sphere_tiny_gaussian", "typed:sphere_tiny_interleaved", "typed:pose3example"],
    ["typed:sphere_small_colamd", "typed:sphere_tiny_cauchy"],
    ["typed:sphere_small_metis", "typed:sphere_tiny_huber", "typed:dubrovnik_3_7_unit", "typed:dubrovnik_3_7_priors"],
    # FP32-storage mode (float instantiations, cp.async staging of floats in the point-leaf Schur kernel)
    ["fp32:bal_tiny_s2", "fp32:bal_tiny_bundler", "fp32:bal_small_metis", "fp32:sphere_tiny_gaussian", "fp32:pose2_ring", "fp32:pose2_ring_colamd",
     "marginals:bal_tiny_s2", "marginals:sphere_tiny", "marginals:bal_tiny_bundler", "marginals:pose2_ring"],
    # degenerate shapes + API misuse; fronts of 128+ columns through both tile-dataflow builds (DMMA fragment layout emulated)
    # ... and long runs of points per CTA (several cp.async batches, both batch sizes, 2 and 3 tiles per thread) in both storage modes
    # coverage: instantiations no fixture reaches (tests/emu/kernel_coverage.py lists what is left)
    ["edge:x", "coverage:x", "midsize:cal3_s2", "midsize:bundler", "midsize:bundler@8", "midsize:cal3_s2@8", "midsize:bundler@4", "midsize:cal3_s2@5", "midsize:bundler@3", "bigfront:x"],
    # the BAL point leaves at mixed separator widths and run lengths (tests/test_point_leaf_shapes.py)
    ["leafshapes:cal3_s2", "leafshapes:bundler"],
    # every allocation of problem creation, Dogleg, joint marginals and the Jacobian storage switch failing in turn: nothing leaks
    ["allocfail:x"],
    # the GaussianFactorGraph level, Dogleg, Gauss-Newton
    ["linear:" + c for c in ("lin_pose2_toy", "lin_pose2_synth", "lin_random_nary", "lin_mixed_hessian", "lin_arity8", "lin_sphere_tiny",
                             "lin_bal_tiny", "lin_singular", "lin_family_sfm2", "lin_family_smart", "lin_family_expr")] +
    ["mirror:x", "dogleg:bal_tiny_s2", "dogleg:sphere_tiny", "dogleg:pose2_ring", "gn:sphere_tiny", "gn:pose2_ring",
     "gnc:bal_tiny_outliers"],     # (gnc:sphere_tiny_outliers passes too: 2 minutes of emulation, not kept in the suite)
]


def _build(lib, extra):
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in ("engine.cu", "symbolic.cpp")] + [os.path.join(EMU, "cuda_fake_runtime.cpp")]
    deps = srcs + [os.path.join(CSRC, f) for f in ("kernels.cuh", "front_df.cuh", "engine.cuh", "factors.cuh", "geometry.cuh", "symbolic.h")] + \
        [os.path.join(EMU, "cuda_emu_full.h"), os.path.join(ROOT, "include", "gtsam_b200.h")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(d) for d in deps):
        return subprocess.Popen(["g++", "-O1", "-std=c++20", "-w", "-fPIC", "-shared", "-DB200_EMULATE"] + extra +
                                ["-x", "c++", "-I/usr/local/cuda/include", "-I", EMU] + srcs + ["-o", lib, "-pthread", "-ldl"], cwd=CSRC)
    return None


@pytest.fixture(scope="module")
def emu_libs():
    """(plain build, ASan build or None, libasan path)"""
    asan_rt = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    have_asan = os.path.isabs(asan_rt) and os.path.exists(asan_rt)
    jobs = [_build(LIB, [])] + ([_build(LIB_ASAN, ["-g", "-fsanitize=address"])] if have_asan else [])
    for j in jobs:
        if j is not None and j.wait() != 0:
            raise RuntimeError("emulation build failed")
    return LIB, (LIB_ASAN if have_asan else None), asan_rt


@pytest.fixture(scope="module")
def emu_lib(emu_libs):
    return emu_libs[0]


SHARDED_WORLDS = (2, 4, 8)


@pytest.fixture(scope="module")
def emu_jobs(emu_libs):
    """Everything that runs against the emulated library is started at once (scenario groups, the ranks of the sharded
    solve, the C++ parity drivers of tests/test_shim_emulation.py): about 12 CPU-minutes, 2-3 minutes on 8 cores."""
    jobs = {}
    emu_lib, asan_lib, asan_rt = emu_libs
    # threads of a block run in a freshly shuffled order between barriers (the sharded jobs below: descending, the C++ jobs: ascending)
    trace = os.path.join(os.path.dirname(emu_lib), "kernel_trace_%d.txt" % os.getpid())   # B200_EMU_TRACE_FILE: kernel launch counts
    for f in os.listdir(os.path.dirname(emu_lib)):      # traces of earlier runs (this one's included)
        if f.startswith("kernel_trace_"):
            os.unlink(os.path.join(os.path.dirname(emu_lib), f))
    genv = dict(os.environ, B200_EMU_ORDER="shuffle:1", B200_EMU_TRACE_FILE=trace)
    if asan_lib:
        genv.update(ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0", LD_PRELOAD=asan_rt)
    for i, g in enumerate(GROUPS):
        jobs["group%d" % i] = subprocess.Popen([sys.executable, os.path.join(EMU, "run_scenarios.py"), asan_lib or emu_lib] + g,
                                               stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=genv)
    # the sharded solve: SHARDED_WORLD emulation processes joined by tests/emu/fake_nccl.cpp (built as libnccl.so.2)
    nccl = os.path.join(os.path.dirname(emu_lib), "libnccl.so.2")
    src = os.path.join(EMU, "fake_nccl.cpp")
    if not os.path.exists(nccl) or os.path.getmtime(nccl) < os.path.getmtime(src):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", src, "-o", nccl, "-lrt", "-pthread"])
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.dirname(emu_lib) + ":" + os.environ.get("LD_LIBRARY_PATH", ""), B200_EMU_TRACE_FILE=trace,
               B200_EMU_ORDER="reverse")     # the ranks run their threads in descending order between barriers
    for world in SHARDED_WORLDS:
        uid = (b"/b200emu_pytest_%d_%d" % (os.getpid(), world)).ljust(128, b"\0").hex()
        for r in range(world):
            jobs["world%d_rank%d" % (world, r)] = subprocess.Popen(
                [sys.executable, os.path.join(EMU, "run_sharded.py"), emu_lib, str(r), str(world), uid], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                text=True, env=env)
    ref = os.path.join(ROOT, "oracle", "_ref")
    if os.path.exists(os.path.join(ref, "shim_parity")):
        g = os.path.join(ROOT, "tests", "golden")
        senv = dict(os.environ, LD_PRELOAD=emu_lib, B200_NO_GRAPH="1")
        shim = {
            "lm_bal": ["shim_parity", os.path.join(g, "bal_tiny_s2.prob.bin"), "30", "0"],
            "lm_bundler": ["shim_parity", os.path.join(g, "bal_tiny_bundler.prob.bin"), "30", "1"],
            "lm_pose2": ["shim_parity", os.path.join(g, "pose2_ring_colamd.prob.bin"), "30", "0"],
            "lm_huber": ["shim_parity", os.path.join(g, "sphere_tiny_huber.prob.bin"), "30", "0"],
            "marg": ["shim_marginals", os.path.join(g, "bal_tiny_s2.prob.bin")],
            "lin_nary": ["shim_linear", "graph", os.path.join(g, "lin_random_nary.lin.bin")],
            "lin_hess": ["shim_linear", "graph", os.path.join(g, "lin_mixed_hessian.lin.bin")],
            "lin_sing": ["shim_linear", "graph", os.path.join(g, "lin_singular.lin.bin")],
            "pose2": ["shim_linear", "pose2", os.path.join(g, "data", "synthetic_pose2.g2o"), "30"],
            "families": ["shim_families", "gpu"],
            "gnc": ["shim_marginals", os.path.join(g, "bal_tiny_outliers.prob.bin"), "1"],   # (sphere_tiny_outliers passes too: 3 minutes)
        }
        for k, a in shim.items():
            jobs["shim_" + k] = subprocess.Popen([os.path.join(ref, a[0])] + a[1:], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=senv)
    results = {}
    for k, p in jobs.items():
        try:
            out, err = p.communicate(timeout=1500)
            results[k] = (p.returncode, out, err)
        except subprocess.TimeoutExpired:
            p.kill()
            results[k] = (-999, "", "timeout")
    results["kernel_trace"] = trace
    return results


def test_whole_library_in_host_emulation(emu_jobs):
    failures = []
    for i, g in enumerate(GROUPS):
        rc, out, err = emu_jobs["group%d" % i]
        done = [l.split()[1] for l in out.splitlines() if l.startswith("EMU_OK")]
        if rc != 0 or done != g:
            failures.append((g, done, err[-800:]))
    assert not failures, failures


def test_every_kernel_of_the_gpu_build_is_reached(emu_jobs):
    """Every __global__ function compiled into libgtsam_b200.so (all template instantiations) is launched by at least one
    emulated scenario that checks its results against the reference / the oracle — no kernel ships unexercised."""
    import re
    lib = os.path.join(ROOT, "gtsam_b200", "libgtsam_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")

    def names(lines):
        out = set()
        for l in lines:
            m = re.search(r"(b200::[a-z0-9_]*_kernel(?:<[^(]*>)?)\(", l)
            if m and "__device_stub" not in l and "__wrapper" not in l:
                out.add(m.group(1))
        return out
    built = names(subprocess.run(["nm", "-C", "--defined-only", lib], capture_output=True, text=True).stdout.splitlines())
    assert len(built) > 100
    built.discard("b200::fp64_peak_kernel")     # a measurement aid (roofline denominators of bench.py), no result to check
    mangled = [l.rsplit(" ", 1)[0] for l in open(emu_jobs["kernel_trace"])]
    reached = names(subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.splitlines())
    assert not sorted(built - reached), sorted(built - reached)


@pytest.mark.parametrize("world", SHARDED_WORLDS)
def test_sharded_solve_in_host_emulation(emu_jobs, world):
    """SURVEY 8(e) at 2 (validated on hardware), 4 and 8 ranks: the sharded solve and LM iterations of six problems (BAL with
    the Schur and a METIS ordering, Bundler cameras, COLAMD-ordered Pose3 and Pose2 graphs, a chain) against the same
    problem solved alone, every rank checking its own view; all-reduces through a shared-memory stand-in for NCCL."""
    for r in range(world):
        rc, out, err = emu_jobs["world%d_rank%d" % (world, r)]
        assert rc == 0 and ("SHARDED_OK %d %d" % (r, world)) in out, (r, out[-600:], err[-600:])
