"""User-written targets and metrics against the registry on C7 (funnel, D = 128, 8192 chains,
10 implicit-leapfrog steps per launch), identical inputs:

  fisher   DiagonalRiemannianMetricSystem: the funnel and its Fisher metric as user sources
           (mb200_implicit_leapfrog_riemannian_user) against the registry FunnelFisherMetric
  scalar   ScalarRiemannianMetricSystem: the funnel and s = 1 + |q|^2 / D as user sources against
           the registry QuadraticScalarMetric

For each: the median of --reps CUDA-event-timed launches after --warmup launches, chain-steps/s,
fixed-point iterations per completed step, the cold NVRTC compile time of the user image, and the
largest relative difference of pos / mom / h to the registry.  Card name, power limit and SM
clock are read in the same run.  Prints one JSON line.

    python profiles/tools/bench_user_riemannian.py [--reps 10] [--warmup 3]
"""

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

from bench_user_target import card, timed  # noqa: E402
from mici_b200 import engine, jit, problems  # noqa: E402
from test_user_riemannian_gpu import user_system  # noqa: E402


def rel(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    ok = np.isfinite(a) & np.isfinite(b)
    return float(np.max(np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-300), initial=0.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    out = {"card": card(), "chains": args.chains, "dim": args.dim, "steps": args.steps}
    for kind in ("fisher", "scalar"):
        prob = problems.make_problem("C7", n_chains=args.chains, dim=args.dim, metric_kind=kind)
        state = engine.build_state(prob, "cuda:0")
        usr = user_system(prob)
        t0 = time.perf_counter()
        usr._user_pair.handle()  # compile (cold: a new source per process) and load
        compile_s = time.perf_counter() - t0
        res = {"compile_s": compile_s}
        news = {}
        for label, system in (("registry", engine.build_system(prob)), ("user", usr)):
            integ = engine.build_integrator(prob, system=system)
            news[label] = integ.step_n(state, args.steps, return_h=True)
            sec = timed(lambda: integ.step_n(state, args.steps), args.reps, args.warmup)
            new = news[label]
            done = new.n_done > 0
            iters = new.solver_iters[done].sum(1).double().mean().item()
            res[label] = {"seconds": sec, "chain_steps_per_s": args.chains * args.steps / sec,
                          "fp_iters_last_step": iters, "completed": int(done.sum())}
        r, u = news["registry"], news["user"]
        res["max_rel_diff"] = max(rel(u.pos, r.pos), rel(u.mom, r.mom), rel(u.h, r.h))
        res["bitwise"] = bool(torch.equal(u.pos, r.pos) and torch.equal(u.mom, r.mom)
                              and torch.equal(torch.nan_to_num(u.h), torch.nan_to_num(r.h)))
        res["user_over_registry"] = res["user"]["chain_steps_per_s"] / res["registry"][
            "chain_steps_per_s"]
        out[kind] = res
    out["nvrtc"] = "%d.%d" % jit.version()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
