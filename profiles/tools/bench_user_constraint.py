"""User-written constraints against the registry on C9 (GaussianDenseConstrainedEuclideanMetricSystem,
multi-sphere C = 8, D = 128, dense metric, Newton projection, 8192 chains), identical inputs:

  user       the multi-sphere as a CudaTarget (mb200_constrained_leapfrog_gaussian_euclidean_user:
             the warp kernel K6 with the user functions staged through shared memory)
  registry   the registry multi-sphere on the same warp kernel
             (mb200_constrained_leapfrog_gaussian_euclidean)

For each: the median of --reps CUDA-event-timed ``step_n`` calls after --warmup calls, and
chain-steps/s; for the user target the cold NVRTC compile time.  Card name, power limit and SM
clock are read in the same run.  Prints one JSON line.

    python profiles/tools/bench_user_constraint.py [--steps 5] [--reps 10] [--warmup 2]
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
from mici_b200 import engine, jit, problems, systems  # noqa: E402
from user_constraint_sources import registry_as_user  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    info = card()
    prob = problems.make_problem("C9", n_chains=args.chains)
    reg = engine.build_integrator(prob)
    target = registry_as_user(reg.system.target)
    t0 = time.perf_counter()
    target.compile()
    compile_s = time.perf_counter() - t0
    usr = engine.build_integrator(prob, system=systems.GaussianDenseConstrainedEuclideanMetricSystem(
        target, metric=reg.system.metric))
    state = engine.build_state(prob, "cuda:0")
    result = {"card": info, "config": "C9", "chains": args.chains, "dim": prob.dim, "n_constr": 8,
              "steps_per_call": args.steps, "nvrtc": "%d.%d" % jit.version(),
              "user_compile_s": compile_s}
    outs = {}
    for key, integ in (("user", usr), ("registry", reg)):
        box = {}

        def go(integ=integ, box=box):
            box["new"] = integ.step_n(state, args.steps, return_h=True)

        t = timed(go, args.reps, args.warmup)
        outs[key] = box["new"]
        result[key] = {"s_per_call": t, "chain_steps_per_s": args.chains * args.steps / t}
    result["user_over_registry_time"] = result["user"]["s_per_call"] / result["registry"]["s_per_call"]
    u, r = outs["user"], outs["registry"]
    assert torch.equal(u.status, r.status) and torch.equal(u.n_done, r.n_done)
    assert torch.equal(u.solver_iters, r.solver_iters)
    result["user_vs_registry_max_rel_diff"] = max(
        float(((a - b).abs() / b.abs().clamp_min(1e-12)).max()) for a, b in
        ((u.pos, r.pos), (u.mom, r.mom), (u.h, r.h)))
    np.testing.assert_allclose(u.pos.cpu().numpy(), r.pos.cpu().numpy(), rtol=1e-9, atol=1e-12)
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
