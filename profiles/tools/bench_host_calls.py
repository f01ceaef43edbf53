"""Host-side cost of the Python call path, at a chain count small enough that it dominates:

  nuts_lockstep/<system>  one lock-step dynamic transition (MultinomialDynamicIntegrationTransition
                          on an integrator without a fused kernel: one batched step per leaf)
  h/<system>, dh_dmom/<system>
                          one ``system.h`` / ``system.dh_dmom`` call

Each entry is the median over --reps of the wall time of --calls back-to-back calls followed
by a device synchronise, divided by --calls, with min and max beside it.  Card name, power limit
and SM clock are read in the same run.  Prints one JSON line.

    python profiles/tools/bench_host_calls.py [--chains 64] [--calls 200] [--reps 7]
"""

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__))]

from bench_user_target import card  # noqa: E402
from mici_b200 import integrators, systems, targets, transitions  # noqa: E402
from mici_b200.states import ChainState  # noqa: E402


def per_call(fn, calls, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) / calls)
    return {"median_us": 1e6 * float(np.median(times)), "min_us": 1e6 * min(times),
            "max_us": 1e6 * max(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=64)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--depth", type=int, default=4)
    args = ap.parse_args()
    info = card()
    dev = torch.device("cuda:0")
    n, dim = args.chains, args.dim
    rng = np.random.default_rng(1)
    a = rng.standard_normal((dim, dim))
    dense = a @ a.T + dim * np.eye(dim)

    def state(on_sphere=False):
        q = rng.standard_normal((n, dim))
        if on_sphere:
            q /= np.linalg.norm(q, axis=1, keepdims=True)
        return ChainState(pos=torch.as_tensor(q, device=dev),
                          mom=torch.as_tensor(rng.standard_normal((n, dim)), device=dev), dir=1)

    euclid = systems.EuclideanMetricSystem(targets.NealFunnel(dim), metric=dense)
    riemann = systems.DiagonalRiemannianMetricSystem(targets.NealFunnel(dim),
                                                     targets.FunnelFisherMetric())
    constr = systems.DenseConstrainedEuclideanMetricSystem(targets.Sphere(dim), metric=dense)
    results = {}
    for name, system, st in (("euclidean_dense", euclid, state()),
                             ("riemannian_diagonal", riemann, state()),
                             ("constrained_sphere", constr, state(on_sphere=True))):
        results[f"h/{name}"] = per_call(lambda s=system, x=st: s.h(x), args.calls, args.reps)
        results[f"dh_dmom/{name}"] = per_call(lambda s=system, x=st: s.dh_dmom(x), args.calls,
                                              args.reps)
    for name, system, integ, st in (
            ("euclidean_bcss2", euclid,
             integrators.BCSSTwoStageIntegrator(euclid, step_size=0.05), state()),
            ("riemannian_implicit_leapfrog", riemann,
             integrators.ImplicitLeapfrogIntegrator(riemann, step_size=0.05), state()),
            ("constrained_sphere", constr,
             integrators.ConstrainedLeapfrogIntegrator(constr, step_size=0.05),
             state(on_sphere=True))):
        tr = transitions.MultinomialDynamicIntegrationTransition(system, integ,
                                                                 max_tree_depth=args.depth)
        assert not tr._fused
        gen = torch.Generator(device=dev)
        gen.manual_seed(3)
        results[f"nuts_lockstep/{name}"] = per_call(
            lambda tr=tr, x=st, g=gen: tr.sample(x, g), max(1, args.calls // 20), args.reps)
    print(json.dumps({"card": info, "chains": n, "dim": dim, "calls": args.calls,
                      "depth": args.depth, "per_call": results}), flush=True)


if __name__ == "__main__":
    main()
