"""Golden vectors for SuGaR's SDF regulariser, produced by EXECUTING the reference's own source.

From frosting_scene/sugar_model.py, the methods `sample_points_in_gaussians`, `get_covariance`, `get_smallest_axis`,
`get_normals`, `get_beta` and `get_field_values` are cut out of class SuGaR with `ast` and bound to a stub model that
holds the activated tensors (points, scaling, quaternions, strengths, knn_idx, beta_mode 'average').  pytorch3d's
quaternion_apply / quaternion_to_matrix / quaternion_invert are stood in by frosting_b200.scenes' restatements.  The
trainer's own lines frosting_trainers/coarse_density_and_dn_consistency.py:744-833 (the field call, the density-mode
estimation loss with use_projection_as_estimation, and the better-normal loss) are read from that file at run time,
dedented and executed with the trainer's default settings.

Run under torch.use_deterministic_algorithms(True), so that the float32 gradients are reproducible.  The draws are
made once, seeded, in float32 as the trainer makes them: `multinomial` then `randn_like`, recorded as the
reference's code calls them.  The field and the losses are then evaluated on those same draws in float64 and in float32
(the float64 run replays the recorded draws: a float64 randn_like would draw other numbers).  Stored per precision:
per-sample density, beta and target, both terms (the per-sample losses' means) and each term's gradients with respect
to points, scaling, quaternions and strengths.

The scene: 300 Gaussians of frosting_b200.scenes.sugar_scene (K = 16, self first), with one thin axis below 1e-8, one
below 1e-6 and one Gaussian moved far from the others (its samples see only itself); 2 000 samples over a mask of about
two thirds of the Gaussians.

    python tests/golden/make_sugar_reg_golden.py        # writes tests/golden/loss_sugar_sdf_reg.npz

The checkout is found as oracle/build_ref.py finds it ($FROSTING_REFERENCE, else `reference/` beside the repository).
"""
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402
from frosting_b200 import scenes                # noqa: E402

P, K, N, SEED = 300, 16, 2000, 20261017
METHODS = ("sample_points_in_gaussians", "get_covariance", "get_smallest_axis", "get_normals", "get_beta",
           "get_field_values")
TRAINER_LINES = (744, 833)          # 1-based, inclusive


def _methods(path):
    src = open(path).read()
    lines = src.splitlines()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "SuGaR")
    out = [textwrap.dedent("\n".join(lines[n.lineno - 1:n.end_lineno])) for n in cls.body
           if isinstance(n, ast.FunctionDef) and n.name in METHODS]
    assert len(out) == len(METHODS), path
    return "\n\n".join(out) + "\n"


class _Torch:
    """torch, except that multinomial and randn_like record their results the first time and replay them (cast to the
    caller's dtype) afterwards."""

    def __init__(self):
        self.record, self.replay = {}, False

    def __getattr__(self, name):
        return getattr(torch, name)

    def _draw(self, name, like, fn):
        if self.replay:
            return self.record[name].to(like.dtype) if like is not None else self.record[name]
        self.record[name] = fn()
        return self.record[name]

    def multinomial(self, *a, **kw):
        return self._draw("multinomial", None, lambda: torch.multinomial(*a, **kw))

    def randn_like(self, t, **kw):
        return self._draw("randn_like", t, lambda: torch.randn_like(t, **kw))


def make_scene():
    sc = scenes.sugar_scene(P, 5, K=K)
    sc["scaling"][7, sc["scaling"][7].argmin()] = 5e-9
    sc["scaling"][8, sc["scaling"][8].argmin()] = 4e-7
    far = 11
    sc["points"][far] += torch.tensor([50.0, 0.0, 0.0])
    others = torch.arange(P)[torch.arange(P) != far][:K - 1]
    sc["knn_idx"][far] = torch.cat([torch.tensor([far]), others])
    g = torch.Generator().manual_seed(1)
    mask = torch.rand(P, generator=g) < 0.66
    mask[[7, 8, far]] = True
    return sc, mask


def main():
    # the CPU scatters of the indexing backward otherwise sum in an order that varies from run to run
    torch.use_deterministic_algorithms(True)
    root = reference_dir()
    model_py = os.path.join(root, "frosting_scene", "sugar_model.py")
    trainer_py = os.path.join(root, "frosting_trainers", "coarse_density_and_dn_consistency.py")
    if not os.path.exists(model_py):
        raise SystemExit(f"{model_py} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    tlines = open(trainer_py).read().splitlines()[TRAINER_LINES[0] - 1:TRAINER_LINES[1]]
    trainer_src = textwrap.dedent("\n".join(tlines)) + "\n"
    ptorch = _Torch()
    ns = {"torch": ptorch, "np": np, "quaternion_apply": scenes.quaternion_apply,
          "quaternion_to_matrix": scenes.quaternion_to_matrix, "quaternion_invert": scenes.quaternion_invert}
    exec(compile(_methods(model_py), model_py, "exec"), ns)
    code = compile(trainer_src, f"{trainer_py}:{TRAINER_LINES[0]}", "exec")

    sc, mask = make_scene()
    save = {k: v.numpy() for k, v in sc.items()}
    save["mask"] = mask.numpy()
    save["seed"] = np.int64(SEED)
    save["n_samples"] = np.int64(N)
    for tag, dtype in (("f32", torch.float32), ("f64", torch.float64)):
        leaves = {k: sc[k].to(dtype).requires_grad_(True) for k in ("points", "scaling", "quaternions", "strengths")}
        model = types.SimpleNamespace(points=leaves["points"], scaling=leaves["scaling"],
                                      quaternions=leaves["quaternions"], strengths=leaves["strengths"],
                                      knn_idx=sc["knn_idx"], n_points=P, device="cpu", beta_mode="average",
                                      binded_to_surface_mesh=False, get_cameras_spatial_extent=lambda: 1.0)
        for name in METHODS:
            setattr(model, name, types.MethodType(ns[name], model))
        torch.manual_seed(SEED)
        ptorch.replay = tag == "f64"
        samples, sample_idx = model.sample_points_in_gaussians(num_samples=N, sampling_scale_factor=1.5, mask=mask,
                                                               probabilities_proportional_to_volume=False)
        env = dict(ns, sugar=model, sdf_samples=samples, sdf_gaussian_idx=sample_idx, iteration=10_000,
                   start_sdf_estimation_from=9_000, start_sdf_better_normal_from=9_000, use_sdf_estimation_loss=True,
                   use_sdf_better_normal_loss=True, enforce_samples_to_be_on_surface=False, sdf_estimation_mode="density",
                   density_threshold=1., density_factor=1., use_projection_as_estimation=True,
                   sample_only_in_gaussians_close_to_surface=False, normalize_by_sdf_std=False,
                   squared_sdf_estimation_loss=False, sdf_better_normal_gradient_through_normal_only=True,
                   sdf_estimation_factor=1., sdf_better_normal_factor=1., loss=0.,
                   CONSOLE=types.SimpleNamespace(print=print))
        exec(code, env)
        est = env["sdf_estimation_loss"].mean()
        nrm = env["sdf_better_normal_loss"].mean()
        fields = env["fields"]
        save[f"{tag}/density"] = fields["density"].detach().numpy()
        save[f"{tag}/beta"] = fields["beta"].detach().numpy()
        save[f"{tag}/target"] = torch.exp(-0.5 * env["sdf_estimation"].pow(2) / fields["beta"].pow(2)).detach().numpy()
        save[f"{tag}/terms"] = np.array([est.item(), nrm.item()])
        for term, value in (("est", est), ("nrm", nrm)):
            gs = torch.autograd.grad(value, list(leaves.values()), allow_unused=True, retain_graph=True)
            for (k, v), g in zip(leaves.items(), gs):
                save[f"{tag}/d{term}_d{k}"] = (torch.zeros_like(v) if g is None else g).numpy()
        if tag == "f32":
            save["idx"] = sample_idx.numpy()
            save["eps"] = ptorch.record["randn_like"].numpy()
    np.savez_compressed(os.path.join(HERE, "loss_sugar_sdf_reg.npz"), **save)
    print(len(save), "arrays", sum(v.nbytes for v in save.values()), "bytes; terms f64", save["f64/terms"],
          "f32", save["f32/terms"])


if __name__ == "__main__":
    main()
