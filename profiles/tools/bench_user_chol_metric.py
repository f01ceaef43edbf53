"""User-written Cholesky-factor metrics on CholeskyFactoredRiemannianMetricSystem (the
triangular-factored policy, K10 / K14), 8192 chains, implicit leapfrog:

  c8_d64/128/200  the quadratic target and factor model of C8 as user sources
                  (mb200_implicit_leapfrog_riemannian_user) against the registry
                  QuadraticCholeskyMetric on identical inputs; registry and user launches
                  alternate.  Each side's layout is reported: the user image keeps two matrices
                  per chain (L and V), so it leaves shared memory above D = 112, the registry
                  (L only) above D = 156
  ar1_66/256      the hierarchical AR(1) model with its closed-form bidiagonal factor, T = 64
                  and 254

For each: the median of --reps CUDA-event-timed launches of --steps steps after --warmup
launches, chain-steps/s, and for C8 the largest relative difference of pos / mom / h to the
registry; the cold NVRTC compile time of each user image.  Card name, power limit and SM clock
are read in the same run.  Prints one JSON line.

    python profiles/tools/bench_user_chol_metric.py [--reps 10] [--warmup 3]
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
from test_user_chol_metric_gpu import user_system  # noqa: E402

import make_user_chol_metric_golden as ul  # noqa: E402


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


RM_SMEM_BYTES = 227 * 1024  # riemannian.cuh: opt-in shared memory per CTA on sm_90


def layout(dim, n_mats):
    """Where the launch plan keeps a chain's matrices: the size rm_carve (riemannian.cuh) gives an
    RM_MATRICES layout with n_mats matrices, against RM_SMEM_BYTES."""
    ld, dpad = dim + 1, (dim + 1) & ~1
    vec = 27 * dpad + 3 * (dpad // 2 + 2) + 40
    return "shared" if (dim * ld * n_mats + vec) * 8 <= RM_SMEM_BYTES else "workspace"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    n = args.chains
    out = {"card": card(), "chains": n, "steps": args.steps, "reps": args.reps}

    # ---- C8: user against registry, alternating launches
    first = True
    for dim in (64, 128, 200):
        prob = problems.make_problem("C8", n_chains=n, dim=dim)
        state = engine.build_state(prob, "cuda:0")
        usr = user_system(prob)
        res = {"layout_registry": layout(dim, 1), "layout_user": layout(dim, 2)}
        if first:
            out["compile_s_quadratic_chol"] = compile_and_load(usr)
            first = False
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
        res["user_over_registry"] = res["user"]["chain_steps_per_s"] / res["registry"][
            "chain_steps_per_s"]
        out[f"c8_d{dim}"] = res
        del integs, news, state
        torch.cuda.empty_cache()

    # ---- the hierarchical AR(1) model at n chains: the fixture case's positions and momenta
    # tiled over the batch
    first = True
    for case in ("ul_ar1_64_leapfrog", "ul_ar1_254_leapfrog"):
        p = ul.case_problem(case)
        reps = -(-n // p.n_chains)
        pos = torch.as_tensor(np.tile(p.pos, (reps, 1))[:n], device="cuda:0")
        mom = torch.as_tensor(np.tile(p.mom, (reps, 1))[:n], device="cuda:0")
        st = ChainState(pos=pos, mom=mom, dir=1)
        system = user_system(p)
        dim = p.pos.shape[1]
        res = {"dim": dim, "layout_user": layout(dim, 2)}
        if first:
            out["compile_s_ar1"] = compile_and_load(system)
            first = False
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
        out[f"ar1_{dim}"] = res
    out["nvrtc"] = "%d.%d" % jit.version()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
