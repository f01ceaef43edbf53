"""User-written targets against the registry on C1 (funnel, D = 128, 8192 chains, dense metric,
50 leapfrog steps per launch), identical inputs:

  user       the funnel as a CudaTarget (mb200_leapfrog_euclidean_user: K1g + shared-memory staging)
  registry   the registry funnel on the same general-dimension kernel K1g
             (mb200_leapfrog_euclidean_generic)
  default    mb200_leapfrog_euclidean, which takes the tensor-core kernel K1 for this shape
  logistic   the logistic-regression user target (200 x 25 design, dense metric), same launch shape

For each: the median of --reps CUDA-event-timed launches after --warmup launches, chain-steps/s,
and for the user targets the cold NVRTC compile time.  Card name, power limit and SM clock are
read in the same run.  Prints one JSON line.

    python profiles/tools/bench_user_target.py [--reps 20] [--warmup 3]
"""

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from mici_b200 import _lib, jit, systems  # noqa: E402
from mici_b200.targets import CudaTarget, NealFunnel  # noqa: E402
from user_target_sources import FUNNEL, logistic  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.splitlines()[0]
    return dict(zip(q.split(","), (s.strip() for s in out.split(","))))


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n, n_steps = args.chains, args.steps
    info = card()
    lib = _lib.load()
    result = {"card": info, "chains": n, "steps_per_launch": n_steps,
              "nvrtc": "%d.%d" % jit.version()}

    def setup(target, eps, seed):
        dim = target.dim
        rng = np.random.default_rng(seed)
        a = rng.normal(size=(dim, dim)) / np.sqrt(dim)
        system = systems.EuclideanMetricSystem(target, metric=a @ a.T + np.identity(dim))
        q = torch.as_tensor(rng.normal(size=(n, dim)) * 0.5, device=dev)
        p = torch.as_tensor(rng.normal(size=(n, dim)), device=dev)
        qo, po = torch.empty_like(q), torch.empty_like(p)
        model = system._model(dev)
        minv = system.metric.inv_device(dev)

        def launcher(entry, user=None):
            extra = () if user is None else (user,)

            def go():
                rc = getattr(lib, entry)(
                    _lib.ptr(q), _lib.ptr(p), _lib.ptr(qo), _lib.ptr(po), None, n, dim, eps, None,
                    n_steps, None, 0, None, 1, 2, _lib.ptr(minv), ctypes.byref(model), None, None,
                    None, _lib.current_stream_ptr(dev), *extra)
                _lib.check(rc, entry)
            return go, qo, po
        return launcher

    def compile_cold(t):
        t0 = time.perf_counter()
        t.compile()
        return time.perf_counter() - t0

    user = CudaTarget(128, FUNNEL, name="funnel")
    result["user_compile_s"] = compile_cold(user)
    outs = {}
    for key, target, entry in (("user", user, "mb200_leapfrog_euclidean_user"),
                               ("registry", NealFunnel(128), "mb200_leapfrog_euclidean_generic"),
                               ("default", NealFunnel(128), "mb200_leapfrog_euclidean")):
        go, qo, po = setup(target, 0.05, 1)(
            entry, target.handle() if isinstance(target, CudaTarget) else None)
        t = timed(go, args.reps, args.warmup)
        outs[key] = (qo.clone(), po.clone())
        result[key] = {"s_per_launch": t, "chain_steps_per_s": n * n_steps / t}
    for key in ("registry", "default"):
        result[f"user_vs_{key}_max_rel_diff"] = max(
            float(((a - b).abs() / b.abs().clamp_min(1e-12)).max()) for a, b in
            zip(outs["user"], outs[key]))
    np.testing.assert_allclose(outs["user"][0].cpu().numpy(), outs["registry"][0].cpu().numpy(),
                               rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(outs["user"][1].cpu().numpy(), outs["registry"][1].cpu().numpy(),
                               rtol=1e-10, atol=1e-12)
    result["user_vs_registry_agree"] = True

    lr = logistic()
    result["logistic_compile_s"] = compile_cold(lr)
    go, _, _ = setup(lr, 0.2, 2)("mb200_leapfrog_euclidean_user", lr.handle())
    t = timed(go, args.reps, args.warmup)
    result["logistic"] = {"dim": lr.dim, "s_per_launch": t, "chain_steps_per_s": n * n_steps / t}
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
