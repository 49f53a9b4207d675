"""Data-parallel sharding of the crop batch over the GPUs of one node (SURVEY.md 8e).

Crops (= persons x test-time augmentations, multiperson_model.py:240) are independent through the backbone, head and
decode, so rank r processes the contiguous chunk ``shard_range(B, world, r)`` with replicated weights.  The only
exchange is ONE all-gather per forward.  Because ``reconstruct_ref_fullpersp`` normalises with batch-global RMS
scalars (ptu3d.py:71-74), the gathered tensor is ``[coords2d | coords3d_rel]`` (5 floats per joint) and every rank
runs the (tiny) absolute reconstruction on the full batch: the sharded result is then identical to the unsharded
reference, not merely within tolerance.  Chunk order = rank order, so the gather is a plain concatenation.  A
latent-point model gathers and reconstructs its latents and maps them to joints after the reconstruction."""
import torch


def shard_range(n, world_size, rank):
    """Contiguous, balanced chunks (first ``n % world`` ranks get one extra crop)."""
    base, rem = divmod(n, world_size)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard_sizes(n, world_size):
    return [shard_range(n, world_size, r)[1] - shard_range(n, world_size, r)[0] for r in range(world_size)]


def pack_decoded(coords2d, coords3d_rel):
    """[b,J,2], [b,J,3] -> [b,J,5] (what travels in the all-gather)."""
    return torch.cat([coords2d, coords3d_rel], dim=-1).contiguous()


def unpack_decoded(packed):
    return packed[..., :2].contiguous(), packed[..., 2:].contiguous()


def gather_decoded(local_packed, n_total, world_size, all_gather_fn):
    """Ragged-safe gather: chunks are padded to the largest shard, gathered, trimmed and concatenated in rank order.
    ``all_gather_fn(tensor) -> [world, *tensor.shape]`` (NCCL through mtb_allgather_joints on the device;
    torch.distributed gloo in the CPU tests)."""
    sizes = shard_sizes(n_total, world_size)
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(local_packed.shape[1:]), dtype=local_packed.dtype, device=local_packed.device)
    pad[:local_packed.shape[0]] = local_packed
    allp = all_gather_fn(pad)
    return torch.cat([allp[r, :sizes[r]] for r in range(world_size)], dim=0)


class ShardedMetrabs:
    """Runs ``model`` (metrabs_b200.models.metrabs.Metrabs) data-parallel: every rank passes the FULL flat crop batch
    (or just its own chunk with ``presharded=True``) and gets the full [B,J,3] result.  ``engine`` (optional) replaces
    ``model.engine(device)``: any object with ``n_joints``, ``backbone``, ``head_decode``, ``allgather``,
    ``reconstruct_absolute`` (and optionally ``forward_sharded``, and ``n_points`` / ``combine_latents`` for a
    latent-point model) - the CPU tests drive the host logic through it."""

    def __init__(self, model, rank, world_size, engine=None):
        self.model, self.rank, self.world, self._engine = model, rank, world_size, engine

    def forward(self, crops, intrinsics, n_total=None, presharded=False):
        eng = self._engine if self._engine is not None else self.model.engine(crops.device)
        if presharded:
            local = crops
        else:
            n_total = crops.shape[0]
            s, e = shard_range(n_total, self.world, self.rank)
            local = crops[s:e]
        sizes = shard_sizes(n_total, self.world)
        if min(sizes) == max(sizes) and sizes[0] > 0 and hasattr(eng, 'forward_sharded'):
            # equal shards: the whole step in one library call on preallocated buffers (mtb_forward_sharded)
            return eng.forward_sharded(local, intrinsics)
        if local.shape[0] == 0:
            # fewer crops than ranks (e.g. 3 person-crops on 8 GPUs): this rank has nothing to compute but must still
            # take part in the collective
            packed_local = torch.zeros((0, getattr(eng, 'n_points', eng.n_joints), 5), dtype=torch.float32,
                                       device=crops.device)
        else:
            feats = eng.backbone(local)
            c2d, c3d = eng.head_decode(feats)
            packed_local = pack_decoded(c2d, c3d)
        packed = gather_decoded(packed_local, n_total, self.world, lambda t: eng.allgather(t).clone())
        g2d, g3d = unpack_decoded(packed)
        out = eng.reconstruct_absolute(g2d, g3d, intrinsics)
        combine = getattr(eng, 'combine_latents', None)
        return combine(out) if combine is not None else out
