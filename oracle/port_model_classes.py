"""TEST INFRASTRUCTURE ONLY - torch-cpu restatement of the reference's two other model classes, ``Metro`` and ``Model25D``.

The reference has both only as TF/Keras code (``metrabs_tf/models/metro.py:13-45``, ``metrabs_tf/models/twofive.py:14-57``,
``metrabs_tf/models/util.py:8-28``, ``metrabs_tf/tfu.py:216-233``, ``metrabs_tf/tfu3d.py:210-269``) and TensorFlow is not part
of this build, so parity is "this build's restatement vs this build's kernels", as for the ResNet and MobileNet ports.  The
backbones, their state dicts and the MeTRAbs pieces come from ``oracle/port.py`` and its siblings unchanged.

Head (``Head3D`` = ``Head25D``): ``conv_final`` 1x1 with bias and ``D*J`` channels, channel ``d*J + j`` (rearrange
``b h w (d j) -> b h w d j``); fp32 soft-argmax jointly over (W, H, D), output (x, y, z), with ``tf.linspace(0, 1, n)``, which is
``[0]`` for ``n == 1``.  Metro: ``heatmap_to_metric``; Model25D: ``heatmap_to_25d`` (x, y image pixels, z mm).  The TF
``heatmap_to_image`` has no ``legacy_centered_stride_bug`` term, so that flag is refused.

``reconstruct_absolute_by_bone_lengths(coords25d, K, L, edges, only_in_fov=True, max_iter=10)``:

1. ``n2d = ([x, y, 1] @ inv(K)^T)[:2]``; ``z_rel = z - mean_j z`` (``mean_relative``) or ``z - z[:, -1]``.
2. ``w_e = (in_fov_i and in_fov_j) + 1e-8`` per bone ``e = (i, j)``, with MeTRAbs' ``is_within_fov`` on the pixel coordinates.
3. ``guess = 1500 / max(max_j n2d - min_j n2d)`` (outer max over x and y).
4. ``x_j = [n2d_j, 1]``, ``a = x_i - x_j``, ``b = x_i z_rel_i - x_j z_rel_j``, ``c = |a|^2``, ``d = 2 a.b``, ``e = |b|^2``;
   residual ``r_e(z) = (sqrt(z^2 c + z d + e) - L_e) w_e``.
5. ``z_ref`` = tensorflow_graphics' ``levenberg_marquardt.minimize(residual_fn, guess[:, None], 10)[1][0][:, 0]``, restated
   (the package is neither vendored nor installed): the minimiser flattens the ``B*E`` residuals into one vector, so its
   Jacobian ``[B*E, B]`` is block-diagonal and ``lstsq(J, r, l2_regularizer=lam)`` is, per crop,
   ``delta_b = sum_e J_be r_be / (sum_e J_be^2 + lam)`` with ``J_be = w_e (2 z c_e + d_e) / (2 sqrt(z^2 c_e + z d_e + e_e))``;
   the candidate ``z - delta`` replaces ``z`` for ALL crops iff the sum of squares over the whole batch decreases, else every
   crop keeps its value and ``lam *= 10``; ``lam`` starts at 1e-20; 10 iterations.
6. ``out = [n2d, 1] * (z_rel + z_ref)``.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import port

HEAD_KEY = 'heatmap_head.conv_final'


def linspace01_tf(n, dtype=torch.float32):
    """tf.linspace(0., 1., n): [0] for n == 1 (ptu.linspace gives [0.5])."""
    return torch.linspace(0.0, 1.0, n, dtype=dtype) if n > 1 else torch.zeros(1, dtype=dtype)


def soft_argmax_tf(logits, dims):
    """tfu.soft_argmax (tfu.py:216-233): joint softmax over ``dims``, per-axis expectation with tf.linspace."""
    dims = tuple(d if d >= 0 else logits.ndim + d for d in dims)
    mx = torch.amax(logits, dim=dims, keepdim=True)
    e = torch.exp(logits - mx)
    p = e / torch.sum(e, dim=dims, keepdim=True)
    out = []
    for d in dims:
        others = [o for o in dims if o != d]
        marg = torch.sum(p, dim=others, keepdim=True)
        shape = [1] * logits.ndim
        shape[d] = logits.shape[d]
        coord = (marg * linspace01_tf(logits.shape[d], logits.dtype).reshape(shape)).sum(dim=d, keepdim=True)
        for hd in sorted(dims, reverse=True):
            coord = coord.squeeze(hd)
        out.append(coord)
    return torch.stack(out, dim=-1)


def _check_cfg(cfg):
    if cfg.legacy_centered_stride_bug:
        raise ValueError('Metro / Model25D decode with the TF heatmap_to_image, which has no legacy_centered_stride_bug term')


def head_heatmap_coords(sd, features, cfg, n_joints, prefix=HEAD_KEY):
    """Head3D up to the soft-argmax: features [B,C,H,W] -> [B,J,3] in [0, 1] heatmap units, order (x, y, z)."""
    _check_cfg(cfg)
    x = F.conv2d(features.float(), sd[prefix + '.weight'], sd[prefix + '.bias'])
    b, _, h, w = x.shape
    logits = x.reshape(b, cfg.depth, n_joints, h, w)  # b (d j) h w -> b d j h w
    return soft_argmax_tf(logits, dims=(4, 3, 1))


def heatmap_to_25d(coords, cfg):
    """metrabs_tf/models/util.py:21-23 (inference: stride_test)."""
    return torch.cat([port.heatmap_to_image(coords[..., :2], cfg), coords[..., 2:] * cfg.box_size_mm], dim=-1)


def metro_head(sd, features, cfg, n_joints):
    """Metro's output: heatmap_to_metric of the head, [B,J,3] mm relative to the crop box."""
    return port.heatmap_to_metric(head_heatmap_coords(sd, features, cfg, n_joints), cfg)


def head_25d(sd, features, cfg, n_joints):
    """Model25D's head: coords25d [B,J,3] = (x px, y px, z mm)."""
    return heatmap_to_25d(head_heatmap_coords(sd, features, cfg, n_joints), cfg)


# ---------------------------------------------------------------------------------------------- the bone-length solve
def bone_problem(coords25d, intrinsics, edges, cfg, mean_relative=True):
    """Steps 1-4: -> (n2d [B,J,2], z_rel [B,J], coef (c, d, e, w) each [B,E], guess [B])."""
    coords25d = coords25d.float()
    inv_k = torch.linalg.inv(intrinsics.float())
    n2d = (port.to_homogeneous(coords25d[..., :2]) @ inv_k.transpose(1, 2))[..., :2]
    z = coords25d[..., 2]
    z_rel = z - (z.mean(dim=1, keepdim=True) if mean_relative else z[:, -1:])
    edges = torch.as_tensor(np.asarray(edges), dtype=torch.long).reshape(-1, 2)
    i, j = edges[:, 0], edges[:, 1]
    in_fov = port.is_within_fov(coords25d[..., :2], cfg)
    w = torch.logical_and(in_fov[:, i], in_fov[:, j]).float() + np.float32(1e-8)
    x = port.to_homogeneous(n2d)
    a = x[:, i] - x[:, j]
    y = x * z_rel[..., None]
    b = y[:, i] - y[:, j]
    c = a.square().sum(-1)
    d = 2 * (a * b).sum(-1)
    e = b.square().sum(-1)
    size = (n2d.amax(dim=1) - n2d.amin(dim=1)).amax(dim=-1)
    return n2d, z_rel, (c, d, e, w), 1500 / size


def bone_residuals(z, coef, lengths):
    c, d, e, w = coef
    z = z[:, None]
    return (torch.sqrt(z.square() * c + z * d + e) - lengths) * w


def bone_jacobian(z, coef):
    c, d, e, w = coef
    z = z[:, None]
    return w * (2 * z * c + d) / (2 * torch.sqrt(z.square() * c + z * d + e))


def levenberg_marquardt(residual_fn, jacobian_fn, z0, max_iter=10, trace=None):
    """The restated minimiser (step 5) for B independent scalars coupled only through the accept decision.
    ``residual_fn(z [B]) -> [B, E]``, ``jacobian_fn(z) -> [B, E]`` (d r / d z of each crop's own z).  ``trace``, a list, gets one
    dict per iteration: candidate, accepted, z after the iteration, objective before and of the candidate, lam used."""
    z = z0.float().clone()
    objective = residual_fn(z).square().sum()
    lam = torch.tensor(1e-20, dtype=torch.float32)
    for _ in range(max_iter):
        r = residual_fn(z)
        jac = jacobian_fn(z)
        candidate = z - (jac * r).sum(dim=1) / (jac.square().sum(dim=1) + lam)
        new_objective = residual_fn(candidate).square().sum()
        accepted = bool(new_objective < objective)
        entry = dict(candidate=candidate, objective=objective, new_objective=new_objective, lam=float(lam),
                     accepted=accepted)
        if accepted:
            z, objective = candidate, new_objective
        else:
            lam = lam * 10
        if trace is not None:
            trace.append(dict(entry, z=z.clone()))
    return z


def reconstruct_by_bone_lengths(coords25d, intrinsics, bone_lengths, edges, cfg, mean_relative=True, max_iter=10, trace=None):
    """tfu3d.reconstruct_absolute_by_bone_lengths: coords25d [B,J,3] + K [B,3,3] -> camera-space joints [B,J,3]."""
    n2d, z_rel, coef, guess = bone_problem(coords25d, intrinsics, edges, cfg, mean_relative)
    lengths = torch.as_tensor(np.asarray(bone_lengths), dtype=torch.float32)
    z_ref = levenberg_marquardt(lambda z: bone_residuals(z, coef, lengths), lambda z: bone_jacobian(z, coef), guess,
                                max_iter, trace)
    return port.to_homogeneous(n2d) * (z_rel + z_ref[:, None])[..., None]


# ---------------------------------------------------------------------------------------------- models and test data
def metro_forward(sd, features_fn, cfg, n_joints, image):
    """Metro.call(image): ``features_fn(sd, image) -> [B,C,H,W]`` (the backbone restatement)."""
    return metro_head(sd, features_fn(sd, image), cfg, n_joints)


def model25d_forward(sd, features_fn, cfg, n_joints, image, intrinsics, bone_lengths, edges, mean_relative=True):
    """Model25D.call((image, intrinsics))."""
    coords25d = head_25d(sd, features_fn(sd, image), cfg, n_joints)
    return reconstruct_by_bone_lengths(coords25d, intrinsics, bone_lengths, edges, cfg, mean_relative)


def to_volumetric_state_dict(sd, n_joints):
    """A MeTRAbs state dict (``heatmap_heads.conv_final``, J + D*J channels) -> the Metro / Model25D schema: the backbone keys
    as they are and ``heatmap_head.conv_final`` = the MeTRAbs head's D*J volumetric channels (same layout d*J + j)."""
    out = {k: v for k, v in sd.items() if not k.startswith('heatmap_heads.')}
    out[HEAD_KEY + '.weight'] = sd['heatmap_heads.conv_final.weight'][n_joints:].clone()
    out[HEAD_KEY + '.bias'] = sd['heatmap_heads.conv_final.bias'][n_joints:].clone()
    return out


def tree_edges(n_joints):
    """A binary-tree stick figure over ``n_joints`` joints: edge (parent(j), j) for j >= 1."""
    return [((j - 1) // 2, j) for j in range(1, n_joints)]


def seeded_bone_lengths(n_bones, seed=0):
    """Ideal bone lengths U[150, 450) mm."""
    g = torch.Generator().manual_seed(3000 + seed)
    return (150 + 300 * torch.rand(n_bones, generator=g)).numpy().astype(np.float32)


def synthetic_pose_25d(batch, n_joints, cfg, seed=0, depth_mm=8000.0):
    """Camera-space poses [B,J,3] (extent ~1.5 m at ``depth_mm``), their intrinsics and their exact 2.5D coordinates
    (pixels by projection, z in mm shifted by an arbitrary per-crop offset that the solve must not see)."""
    g = torch.Generator().manual_seed(4000 + seed)
    pose = (torch.rand(batch, n_joints, 3, generator=g) - 0.5) * torch.tensor([800.0, 1500.0, 600.0])
    pose[..., 2] += depth_mm + 1000 * torch.rand(batch, 1, generator=g)
    f = 900 + 200 * torch.rand(batch, generator=g)
    k = torch.zeros(batch, 3, 3)
    k[:, 0, 0] = f
    k[:, 1, 1] = f
    k[:, 0, 2] = cfg.proc_side / 2
    k[:, 1, 2] = cfg.proc_side / 2
    k[:, 2, 2] = 1
    proj = pose @ k.transpose(1, 2)
    px = proj[..., :2] / proj[..., 2:]
    z = pose[..., 2:] - 0.5 * cfg.box_size_mm * torch.rand(batch, 1, 1, generator=g) - depth_mm
    return pose, k, torch.cat([px, z], dim=-1)


def bone_lengths_of(pose, edges):
    """[J,3] pose -> [E] bone lengths."""
    e = torch.as_tensor(np.asarray(edges), dtype=torch.long)
    return (pose[e[:, 0]] - pose[e[:, 1]]).norm(dim=-1)

