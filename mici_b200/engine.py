"""Build (system, integrator, state) on a device from a ``problems.Problem`` description."""

from __future__ import annotations

import torch

from . import integrators, systems, targets
from .states import ChainState


def build_system(problem):
    target = targets.make_target(problem.target, **problem.target_params)
    if problem.system == "euclidean":
        return systems.EuclideanMetricSystem(target, metric=problem.metric)
    if problem.system == "gaussian_euclidean":
        return systems.GaussianEuclideanMetricSystem(target, metric=problem.metric)
    if problem.system == "constrained_euclidean":
        return systems.DenseConstrainedEuclideanMetricSystem(
            target, target, metric=problem.metric,
            dens_wrt_hausdorff=problem.system_kwargs.get("dens_wrt_hausdorff", True))
    if problem.system == "gaussian_constrained_euclidean":
        return systems.GaussianDenseConstrainedEuclideanMetricSystem(
            target, target, metric=problem.metric)
    if problem.system == "softabs_riemannian":
        return systems.SoftAbsRiemannianMetricSystem(target, **problem.system_kwargs)
    if problem.system == "dense_riemannian":
        mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
        return systems.DenseRiemannianMetricSystem(target, mm)
    if problem.system == "diagonal_riemannian":
        mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
        return systems.DiagonalRiemannianMetricSystem(target, mm)
    if problem.system == "scalar_riemannian":
        mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
        return systems.ScalarRiemannianMetricSystem(target, mm)
    if problem.system == "cholesky_riemannian":
        mm = targets.make_metric_model(problem.metric_model, **problem.metric_params)
        return systems.CholeskyFactoredRiemannianMetricSystem(target, mm)
    raise KeyError(problem.system)


def build_integrator(problem, system=None, **overrides):
    system = build_system(problem) if system is None else system
    kw = dict(problem.integrator_kwargs)
    kw.update(overrides)
    if isinstance(kw.get("fixed_point_solver"), str):  # solver named by string in the fixtures
        from . import solvers  # noqa: PLC0415

        kw["fixed_point_solver"] = getattr(solvers, "solve_fixed_point_" + kw["fixed_point_solver"])
    if isinstance(kw.get("projection_solver"), str):
        from . import solvers  # noqa: PLC0415

        kw["projection_solver"] = getattr(
            solvers, "solve_projection_onto_manifold_" + kw["projection_solver"])
    cls = {
        "leapfrog": integrators.LeapfrogIntegrator,
        "implicit_leapfrog": integrators.ImplicitLeapfrogIntegrator,
        "constrained_leapfrog": integrators.ConstrainedLeapfrogIntegrator,
        "implicit_midpoint": integrators.ImplicitMidpointIntegrator,
        "bcss2": integrators.BCSSTwoStageIntegrator,
        "bcss3": integrators.BCSSThreeStageIntegrator,
        "bcss4": integrators.BCSSFourStageIntegrator,
    }[problem.integrator]
    return cls(system, problem.step_size, **kw)


def build_state(problem, device="cuda", dirs=None, chains=None):
    sl = slice(None) if chains is None else chains
    pos = torch.as_tensor(problem.pos[sl], dtype=torch.float64).to(device).contiguous()
    mom = torch.as_tensor(problem.mom[sl], dtype=torch.float64).to(device).contiguous()
    if dirs is None:
        d = 1
    else:
        d = torch.as_tensor(dirs, dtype=torch.int32).to(device)
    return ChainState(pos=pos, mom=mom, dir=d)
