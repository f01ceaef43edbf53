"""User-written dense metrics on DenseRiemannianMetricSystem (the global-workspace dense policy),
8192 chains, implicit leapfrog:

  c5         the quadratic target and the Hadamard metric of C5 at D = 512 as user sources
             (mb200_implicit_leapfrog_riemannian_user) against the registry HadamardMetric on its
             generic rank-one route (generic_rank1_vjp=True: the same V = -w w^T VJP), identical
             inputs; registry and user launches alternate
  logistic   Bayesian logistic regression with its dense Fisher metric, D = 25, 40 rows
  lgcp64     the log-Gaussian Cox process metric C^-1 + diag(m e^x), D = 64
  lgcp144    the same at D = 144

For each: the median of --reps CUDA-event-timed launches of --steps steps after --warmup
launches, chain-steps/s, the cold NVRTC compile time of the user image, and for c5 the largest
relative difference of pos / mom / h to the registry.  Card name, power limit and SM clock are
read in the same run.  Prints one JSON line.

    python profiles/tools/bench_user_dense_metric.py [--reps 10] [--warmup 3]
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

from bench_user_target import card  # noqa: E402
from mici_b200 import engine, jit, problems  # noqa: E402
from mici_b200.states import ChainState  # noqa: E402
from test_user_dense_metric_gpu import user_system  # noqa: E402

import make_user_dense_metric_golden as ud  # noqa: E402


def rel(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    ok = np.isfinite(a) & np.isfinite(b)
    return float(np.max(np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-300), initial=0.0))


def event_time(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3


def compile_and_load(system):
    t0 = time.perf_counter()
    system._user_pair.handle()  # compile (cold: a new source per process) and load
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    n = args.chains
    out = {"card": card(), "chains": n, "steps": args.steps, "reps": args.reps}

    # ---- C5 at D = 512: user against the registry generic route, alternating launches
    prob = problems.make_problem("C5", n_chains=n, dim=512)
    prob.metric_params = dict(prob.metric_params, generic_rank1_vjp=True)
    state = engine.build_state(prob, "cuda:0")
    usr = user_system(prob)
    res = {"compile_s": compile_and_load(usr)}
    integs = {"registry": engine.build_integrator(prob, system=engine.build_system(prob)),
              "user": engine.build_integrator(prob, system=usr)}
    news = {k: i.step_n(state, args.steps, return_h=True) for k, i in integs.items()}
    times = {k: [] for k in integs}
    for rep in range(args.warmup + args.reps):
        for k, integ in integs.items():
            t = event_time(lambda integ=integ: integ.step_n(state, args.steps))
            if rep >= args.warmup:
                times[k].append(t)
    for k in integs:
        sec = float(np.median(times[k]))
        done = news[k].n_done > 0
        res[k] = {"seconds": sec, "chain_steps_per_s": n * args.steps / sec,
                  "completed": int(done.sum()),
                  "fp_iters_last_step": news[k].solver_iters[done].sum(1).double().mean().item()}
    r, u = news["registry"], news["user"]
    res["max_rel_diff"] = max(rel(u.pos, r.pos), rel(u.mom, r.mom), rel(u.h, r.h))
    res["pos_mom_bitwise"] = bool(torch.equal(u.pos, r.pos) and torch.equal(u.mom, r.mom))
    res["user_over_registry"] = res["user"]["chain_steps_per_s"] / res["registry"][
        "chain_steps_per_s"]
    out["c5_d512"] = res
    del integs, news, state
    torch.cuda.empty_cache()

    # ---- models the registry cannot express, at n chains: positions and momenta of the fixture
    # case tiled over the batch
    for model, case in (("logistic", "ud_lr_leapfrog"), ("lgcp64", "ud_lgcp64_leapfrog"),
                        ("lgcp144", "ud_lgcp144_leapfrog")):
        p = ud.case_problem(case)
        reps = -(-n // p.n_chains)
        pos = torch.as_tensor(np.tile(p.pos, (reps, 1))[:n], device="cuda:0")
        mom = torch.as_tensor(np.tile(p.mom, (reps, 1))[:n], device="cuda:0")
        st = ChainState(pos=pos, mom=mom, dir=1)
        system = user_system(p)
        res = {"dim": p.pos.shape[1], "compile_s": compile_and_load(system)}
        integ = engine.build_integrator(p, system=system)
        new = integ.step_n(st, args.steps, return_h=True)
        ts = []
        for rep in range(args.warmup + args.reps):
            t = event_time(lambda: integ.step_n(st, args.steps))
            if rep >= args.warmup:
                ts.append(t)
        sec = float(np.median(ts))
        res.update(seconds=sec, chain_steps_per_s=n * args.steps / sec,
                   completed=int((new.n_done == args.steps).sum()))
        out[model] = res
    out["nvrtc"] = "%d.%d" % jit.version()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
