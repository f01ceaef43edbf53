"""Per-launch CUDA-event times of C9 (GaussianDenseConstrainedEuclideanMetricSystem, multi-sphere
C = 8, D = 128, dense metric, 8192 chains, Newton projection, 10 steps per launch), Newton
iterations per step, the same inputs under DenseConstrainedEuclideanMetricSystem
(dens_wrt_hausdorff=False) in the same process (a different Hamiltonian: the drift is q += dt M^-1 p
and h2 has no q.q/2 term, so not a like-for-like comparison), plus the reference's CPU rate per
core on C9.  Prints one JSON line.
Usage: python profiles/tools/bench_gaussian_constrained.py [--chains N] [--launches K]
       [--ref-chains R]  (--ref-chains 0 skips the reference)"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from mici_b200 import engine, problems  # noqa: E402

N_STEPS = 10


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.splitlines()[0]
    return dict(zip(q.split(","), (x.strip() for x in out.split(","))))


def bench_gpu(config, n_chains, launches, lebesgue_plain=False):
    prob = problems.make_problem(config, n_chains=n_chains)
    if lebesgue_plain:
        prob.system = "constrained_euclidean"
        prob.system_kwargs = {"dens_wrt_hausdorff": False}
    integ = engine.build_integrator(prob)
    state = engine.build_state(prob, "cuda:0")
    for _ in range(2):  # warm-up: module load, occupancy queries
        integ.step_n(state, N_STEPS)
    torch.cuda.synchronize()
    times = []
    for _ in range(launches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        integ.step_n(state, N_STEPS)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    integ.count_calls()
    out = integ.step_n(state, N_STEPS)
    torch.cuda.synchronize()
    steps = float(out.n_done.sum())
    iters = float(integ.call_counts[:, 3].sum())
    med = float(np.median(times))
    return {"config": config, "dim": prob.dim, "chains": n_chains, "steps_per_launch": N_STEPS,
            "ms": [round(t, 4) for t in times], "median_ms": med,
            "steps_per_s": steps / (med * 1e-3), "newton_iters_per_step": iters / steps,
            "complete": float((out.status == 0).double().mean())}


def bench_reference(n_chains):
    """Chain-steps per second of the unmodified reference on one core (oracle/_ref) on C9."""
    import gaussian_constrained_cases as gc
    from oracle import drivers as dr

    if n_chains <= 0 or not dr.reference_available():
        return None
    prob = problems.make_problem("C9", n_chains=n_chains)
    with gc.patched_drivers():
        t = time.perf_counter()
        out = dr.reference_run(prob, N_STEPS)
        dt = time.perf_counter() - t
    return float(out["n_done"].sum()) / dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--ref-chains", type=int, default=8)
    args = ap.parse_args()
    rec = {"bench": "C9 constrained leapfrog, Gaussian split, multi-sphere C=8 D=128, dense metric",
           "gpu": gpu_info()}
    rec["C9"] = bench_gpu("C9", args.chains, args.launches)
    rec["C9"]["reference_cpu_steps_per_s_per_core"] = bench_reference(args.ref_chains)
    rec["C9_inputs_plain_lebesgue_system_different_hamiltonian"] = bench_gpu(
        "C9", args.chains, args.launches, lebesgue_plain=True)
    rec["gpu_after"] = gpu_info()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
