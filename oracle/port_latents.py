"""TEST INFRASTRUCTURE ONLY - CPU restatement of the latent-point MeTRAbs models (affine-combining autoencoder heads),
built on the functions of ``oracle/port.py``.  Like that file it is the checker for the CUDA path, never the product.

It restates what the reference computes with ``affine_weights`` and ``transform_coords`` / ``predict_all_and_latents``
(``/root/reference/metrabs_pytorch/models/metrabs.py`` :23-45, :53-62), with the ``latent_points_to_joints`` that only
the TF model defines (``/root/reference/metrabs_tf/models/metrabs.py`` :80-87 -> ``tfu3d.linear_combine_points``,
``metrabs_tf/tfu3d.py`` :48-49).  Pinned to the unmodified reference by ``tests/golden/latents_tiny_s64.npz``
(``oracle/gen_golden_latents.py``), checked by ``tests/test_oracle_latents.py``.
"""
import torch

from oracle import port


def linear_combine_points(points, weights):
    """metrabs_tf/tfu3d.py:48-49: [B,j,3] x [j,J] -> [B,J,3]."""
    return torch.einsum('bjc,jJ->bJc', points, weights)


def metrabs_forward(sd, spec, cfg: port.PathConfig, n_raw_points, image, intrinsics, w2, n_latents, stages=None):
    """Metrabs.forward of a latent-point model -> joints [B,J,3] fp32: the head over all ``n_raw_points`` points, keep
    points [0, n_latents) (models/metrabs.py:53-55), reconstruct them, then ``einsum('bjc,jJ->bJc', abs, w2)``.
    ``stages`` (dict) receives features, coords2d, coords3d_rel (all ``n_raw_points`` points) and latents_abs."""
    features = port.effnet_features(sd, spec, image)
    coords2d, coords3d_rel = port.heads(sd, features, cfg, n_raw_points)
    latents_abs = port.reconstruct_absolute(coords2d[:, :n_latents], coords3d_rel[:, :n_latents], intrinsics, cfg)
    if stages is not None:
        stages.update(features=features, coords2d=coords2d, coords3d_rel=coords3d_rel, latents_abs=latents_abs)
    return linear_combine_points(latents_abs, torch.as_tensor(w2, dtype=latents_abs.dtype))


def make_affine_weights(n_joints, n_latents, seed=0):
    """Synthetic stand-in for an affine-combining autoencoder file (``--affine-weights``; the real tables are not
    distributed with the code): encoder w1 [J,L] and recombination w2 [L,J], every column summing to 1 (affine
    combinations, as the autoencoder's are), so recombined joints stay in metric range.  Deterministic from the seed;
    float32 numpy."""
    g = torch.Generator().manual_seed(5000 + seed)
    w1 = torch.rand(n_joints, n_latents, generator=g, dtype=torch.float64) + 0.05
    w2 = torch.rand(n_latents, n_joints, generator=g, dtype=torch.float64) + 0.05
    w1 = w1 / w1.sum(dim=0, keepdim=True)
    w2 = w2 / w2.sum(dim=0, keepdim=True)
    return w1.float().numpy(), w2.float().numpy()
