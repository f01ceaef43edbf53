"""Per-launch CUDA-event times of C7 (funnel D = 128, 8192 chains, implicit leapfrog, 10 steps per
launch) with the diagonal Fisher metric and with the scalar metric, plus the reference's CPU
rate per core on the same host.  Prints one JSON line.
Usage: python profiles/tools/bench_diag_riemannian.py [--chains N] [--launches K] [--ref-chains R]"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def bench_gpu(kind, n_chains, launches):
    prob = problems.make_problem("C7", n_chains=n_chains, metric_kind=kind)
    integ = engine.build_integrator(prob)
    state = engine.build_state(prob, "cuda:0")
    for _ in range(2):  # warm-up: module load, occupancy queries
        integ.step_n(state, N_STEPS)
    torch.cuda.synchronize()
    times = []
    for _ in range(launches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = integ.step_n(state, N_STEPS)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    integ.count_calls()
    out = integ.step_n(state, N_STEPS)
    torch.cuda.synchronize()
    steps = float(out.n_done.sum())
    iters = float(integ.call_counts[:, 3].sum())
    med = float(np.median(times))
    return {"metric": kind, "chains": n_chains, "steps_per_launch": N_STEPS, "ms": times,
            "median_ms": med, "steps_per_s": steps / (med * 1e-3),
            "fp_iters_per_step": iters / steps,
            "complete": float((out.status == 0).double().mean())}


def bench_reference(kind, n_chains):
    """Chain-steps per second of the unmodified reference on one core (oracle/_ref)."""
    import riemannian_diag_cases as rc
    from oracle import drivers as dr

    if not dr.reference_available():
        return None
    prob = problems.make_problem("C7", n_chains=n_chains, metric_kind=kind)
    with rc.patched_drivers():
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
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    rec = {"bench": "C7 implicit leapfrog, funnel D=128", "gpu": gpu_info()}
    for kind in ("fisher", "scalar"):
        r = bench_gpu(kind, args.chains, args.launches)
        r["reference_cpu_steps_per_s_per_core"] = bench_reference(kind, args.ref_chains)
        rec[kind] = r
    rec["gpu_after"] = gpu_info()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
