"""GPU: a crop's features, decoded coordinates and joints do not depend on the batch it runs in or where it sits there.

No kernel of the forward makes a crop's value depend on the batch: the kernels are chosen at weight finalization, before
any batch exists; the split-K factor of the SE fc layers depends on channel counts only; every GEMM keeps a fixed K order
per output element; pooling sums each crop in a fixed order.  So ``backbone`` and ``head_decode`` on any contiguous
sub-batch ``crops[s:e]`` (the slice itself, so the pointer offsets are exercised too) must give rows [s, e) of the anchor
batch's results bit for bit (``torch.equal``).  That carries the fp64 checks of test_gpu_forward_ops16.py and
test_gpu_forward_ops32.py, made at their anchor batch, over to every batch and shard: the batch tails below are where a
tile, crop group or partial slice meets the end of the batch.

The one intended batch dependence is the absolute reconstruction, which normalises with batch-global RMS scalars
(ptu3d.py:71-74, recon_pass1_kernel): ``forward`` on a sub-batch must equal ``reconstruct_absolute`` on that sub-batch's
own decode, and it must differ from the anchor's rows for some sub-batch (the sensitivity control).

Per configuration and mode:
* sub-batches: prefixes, every shard of ``parallel.shard_range(N, W, r)`` for W = 2, 4, 8, the ragged shards of
  ``shard_range(N - 1, 8, r)``, single crops at 0, 1, 3, 4, N/2, N - 1, and the anchor plus one extra crop;
* the batch tails those sub-batches reach (asserted against TAILS): a flat (mode-0) tensor-core GEMM with B*H*W % 128 != 0,
  one of them with the SE scale in the GEMM; a TMA depthwise op with B % G != 0 (G crops per item); a fused head with
  B % cpt != 0 (cpt crops per tile); an SE fc with B % 64 != 0 (conv_igemm_kernel's row tile); an fmb_kernel launch with an
  odd tile count;
* guard bands: ``forward`` into a prefix view of a NaN-filled buffer leaves the rows behind it alone, and a forward of b
  crops on a larger workspace leaves the bytes past ``mtb_workspace_bytes(b)`` alone;
* parallel.ShardedMetrabs.forward for W = 2, 4, 8 with every rank simulated on this device (an engine adapter whose
  all-gather runs the other ranks' shards through the same engine): equal and ragged shards and fewer crops than ranks,
  every rank bit-equal to ``forward`` on the whole batch;
* the benchmark and latent-point models also through ``forward_sharded`` on a world-size-1 NCCL communicator, and the
  benchmark model through the pipelined host path with two different batches on the two slots.

On a difference the failure names the first backbone op whose rows differ (debug_run_ops on both batches)."""
import time
import types

import numpy as np
import pytest
import torch

from metrabs_b200 import _lib, parallel
from oracle import port
from tests.test_gpu_ops16_vs_conv2d import H, dw_plan  # noqa: F401  (H: the fixture)

pytestmark = pytest.mark.gpu

MODES = ['bf16', 'fp16', 'tf32x3', 'fp32']
# configuration -> bench.build_model arguments (None: built otherwise, see make_model) and anchor batch
CONFIGS = {
    'bench': (dict(size='l', side=256, joints=24), 256),              # bench.py: EfficientNetV2-L@256, 8x8 final map
    'c3': (dict(size='l', side=384, joints=24), 256),                 # EfficientNetV2-L@384, 12x12 final map
    'c4': (dict(size='s', side=256, joints=122), 64),                 # EfficientNetV2-S@256, 1098 head channels: 9 M tiles
    'c2': (None, 128),                                                # ResNet-50, output stride 8, D = 32
    'b0@224': (None, 128),                                            # EfficientNet-B0@224: 7x7 final map, P = 49
    'latent': (None, 128),                                            # test_gpu_latents.py's tiny latent-point model
    'l@64': (dict(size='l', side=64, joints=24), 64),                 # EfficientNetV2-L@64: one fmb tile per crop at 8x8
}
T16 = ('bf16', 'fp16')
# The batch tails each configuration must reach in the 16-bit tensor-core modes (T16) and in 'tf32x3'.  'fp32' runs
# conv_igemm_kernel on every conv and the generic depthwise kernel, so only the SE fc tail applies there.
# - 'tc0': a flat tensor-core GEMM with a partial last row tile; 'tc0+se' the same with the SE scale in the GEMM (se_rows in
#   the 16-bit modes, the A-tile split in 'tf32x3').  ResNet-50 at stride 8 has 64x64 and 32x32 maps only: B*H*W is a
#   multiple of 128 at every batch.  In the 16-bit modes EfficientNetV2-L@256 scales in the GEMM only the projections of at
#   most 256 channels (tc_se_in_gemm), which sit on 16x16 maps (256 rows per crop); its 8x8 ones run se_scale_kernel first.
# - 'dw': the TMA depthwise kernel with a partial crop group.  It groups crops on maps of 8x8 and less (mtb_debug_dw_plan:
#   G = 4 at 8x8 and 7x7, 8 below); c3's 24x24 and 12x12 maps take one crop per item.  ResNet-50 has no depthwise convs.
# - 'head': a fused head with a partial group of crops.  c3's 12x12 map packs one crop per tile (cpt = 1) and ResNet-50's
#   32x32 map whole 256-pixel tiles of one crop (cpt = 0); B0's 7x7 map has no fused plan at all (the unfused head).
# - 'se': an SE fc whose batch is not a multiple of its 64-row tile; ResNet-50 has no squeeze-excitation.
# - 'fmb': an fmb_kernel launch over an odd number of 16x8 tiles.  Only EfficientNetV2-L@64 has a fused stage with an odd
#   tile count per crop (8x8: one tile); the fused stages of the others have 2 tiles or more per crop (16x16 maps and up;
#   at 384 px 48x48 = 3x6 and 96x96 = 6x12), and B0 has no FusedMBConv blocks.
TAILS = {
    'bench': ({'tc0', 'dw', 'head', 'se'}, {'tc0', 'tc0+se', 'se'}),
    'c3': ({'tc0', 'tc0+se', 'se'}, {'tc0', 'tc0+se', 'se'}),
    'c4': ({'tc0', 'tc0+se', 'dw', 'head', 'se'}, {'tc0', 'tc0+se', 'se'}),
    'c2': (set(), set()),
    'b0@224': ({'tc0', 'tc0+se', 'dw', 'se'}, {'tc0', 'tc0+se', 'se'}),
    'latent': ({'tc0', 'tc0+se', 'dw', 'head', 'se'}, {'tc0', 'tc0+se', 'se'}),
    'l@64': ({'tc0', 'tc0+se', 'dw', 'head', 'se', 'fmb'}, {'tc0', 'tc0+se', 'se'}),
}
TC_FLAT = (_lib.TC_CONV, _lib.TC_CONV_SE, _lib.SE_SCALE_TC_CONV, _lib.TC32)


@pytest.fixture(scope='module')
def affine_path(tmp_path_factory):
    from tests import test_gpu_latents as TL
    path = str(tmp_path_factory.mktemp('affine') / 'affine_tiny.npz')
    np.savez(path, w1=TL.G['w1'], w2=TL.G['w2'])
    return path


_WEIGHTS = {}  # configuration -> (PathConfig, state dict), shared by the modes


def make_model(H, config, precision, affine_path):
    """-> (Metrabs model on cuda:0, crop side)"""
    args, _ = CONFIGS[config]
    if args is not None:
        import bench
        a = types.SimpleNamespace(stride=32, depth=8, **args, precision=precision)
        return bench.build_model(a, torch.device('cuda')), a.side
    if config == 'latent':
        from tests import test_gpu_latents as TL
        return TL.latent_model('predict_all_and_latents', precision, affine_path)[0], TL.S
    if config == 'c2':
        # the oracle's calibrated weights (as test_gpu_forward_ops16.py): bench's conditioned random init takes ResNet-50's
        # activations past the fp16 range
        from oracle import port_tf_backbones as tfb
        if config not in _WEIGHTS:
            pcfg = port.PathConfig(proc_side=256, stride_test=8, depth=32)
            _WEIGHTS[config] = pcfg, tfb.make_state_dict(tfb.ResNet50Spec(pcfg), pcfg, 24, seed=0, calib_batch=1)
        pcfg, sd = _WEIGHTS[config]
        return H.device_model_tf('resnet50', pcfg, 24, sd, precision=precision), 256
    from tests import test_gpu_effnet_b as TB
    if config not in _WEIGHTS:
        pcfg, _spec, sd = TB.model('efficientnet-b0', 224, j=24)
        _WEIGHTS[config] = pcfg, sd
    pcfg, sd = _WEIGHTS[config]
    return TB.device_model(H, 'efficientnet-b0', pcfg, 24, sd, precision), 224


def sub_batches(n):
    """[(s, e)]: prefixes, the shards of shard_range(n, W, r) for W = 2, 4, 8 and of shard_range(n - 1, 8, r), single
    crops at 0, 1, 3, 4, n/2, n - 1 (all within the anchor's n crops; the anchor plus one crop is checked separately)."""
    prefixes = sorted({p for p in (1, 2, 3, 31, 32, 33, 97, 129, 255) if p < n} | {n - 1})
    out = [(0, p) for p in prefixes]
    out += [parallel.shard_range(n, w, r) for w in (2, 4, 8) for r in range(w)]
    out += [parallel.shard_range(n - 1, 8, r) for r in range(8)]
    out += [(i, i + 1) for i in (0, 1, 3, 4, n // 2, n - 1)]
    seen, uniq = set(), []
    for se in out:
        if se not in seen and se[1] > se[0]:
            seen.add(se)
            uniq.append(se)
    return uniq


def head_cpt(P):
    """crops per fused head tile (tc_head_plan, csrc/tc_gemm.cuh): 0 for whole 256-pixel tiles of one crop, None without
    a fused plan"""
    if P <= 256:
        return next((c for c in range(256 // P, 0, -1) if c * P % 16 == 0), None)
    return 0 if P % 256 == 0 else None


def tails_reached(eng, precision, batches, fused_head):
    """-> (batch tails reached by these batch sizes, what was seen: TMA crop groups, head cpt, fmb tiles per crop)"""
    lib = _lib.lib()
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    names = eng.op_names()
    reached, seen = set(), {'G': set(), 'fmb tiles/crop': set()}
    for k, nm in enumerate(names):
        io = eng.op_io(k)
        kern = eng.op_kernel(k)
        (hi, wi, cin), (ho, wo, cout) = io['in_shape'], io['out_shape']
        if nm.endswith(('.fc1', '.fc2')):  # conv_igemm_kernel: 128-row tiles from 128 * SMs rows, 64-row tiles below
            reached |= {'se' for b in batches if b % (128 if b >= 128 * sms else 64)}
        elif k > 0 and eng.op_is_fused_block(k - 1):
            continue  # the projection of a fused block runs inside fmb_kernel
        elif eng.op_is_fused_block(k):
            per_crop = -(-wo // 16) * -(-ho // 8)  # 16x8 spatial tiles
            seen['fmb tiles/crop'].add(per_crop)
            reached |= {'fmb' for b in batches if b * per_crop % 2}
        elif kern in TC_FLAT:
            taps = lib.mtb_op_weight_bytes(eng._h, k) / (cin * cout) / (4 if kern == _lib.TC32 else 2)
            if taps == 1 and (hi, wi) == (ho, wo):  # 1x1 stride 1: the flat mode, B*H*W rows in tiles of 128
                tail = [b for b in batches if b * ho * wo % 128]
                reached |= {'tc0' for _ in tail[:1]}
                if tail and (kern == _lib.TC_CONV_SE or (kern == _lib.TC32 and io['scale'])):
                    reached.add('tc0+se')
        elif kern == _lib.DW_TMA:
            g = dw_plan(ho, wo)[0]
            seen['G'].add(g)
            reached |= {'dw' for b in batches if b % g}
    if fused_head:
        cpt = head_cpt(eng.feature_side ** 2)
        seen['cpt'] = cpt
        reached |= {'head' for b in batches if cpt and b % cpt}
    return reached, seen


def first_differing_op(eng, crops, s, e):
    """-> 'op k name: rows [...]' of the first backbone op whose output on crops[s:e] differs from rows [s, e) of its output
    on crops (debug_run_ops on both; the partial pooling slices of the fused SE pools are laid out by batch, skipped)"""
    names = eng.op_names()
    ks = [k for k, nm in enumerate(names) if not nm.endswith('.avgpool')]

    def rows(k):
        a = eng.debug_run_ops(crops, k + 1)[s:e]
        b = eng.debug_run_ops(crops[s:e], k + 1)
        return torch.nonzero((a != b).flatten(1).any(1)).flatten().tolist()
    lo, hi = 0, len(ks) - 1
    if not rows(ks[hi]):
        return 'no backbone op differs'
    while lo < hi:  # the first differing op: the later ones read its output
        mid = (lo + hi) // 2
        if rows(ks[mid]):
            hi = mid
        else:
            lo = mid + 1
    r = rows(ks[lo])
    return f'op {ks[lo]} {names[ks[lo]]}: rows {[s + i for i in r[:16]]}{" ..." if len(r) > 16 else ""} of [{s}, {e})'


class SimulatedRanks:
    """Engine adapter for parallel.ShardedMetrabs on one device: the real engine's stages, no forward_sharded, and an
    all-gather that puts this rank's padded chunk in its slot and runs every other rank's shard through the same engine
    (memoised in ``decoded``), as the other ranks would."""

    def __init__(self, eng, crops, rank, world, decoded):
        self.eng, self.crops, self.rank, self.world, self.decoded = eng, crops, rank, world, decoded
        self.n_joints, self.n_points = eng.n_joints, eng.n_points

    def backbone(self, crops):
        return self.eng.backbone(crops)

    def head_decode(self, feats):
        return self.eng.head_decode(feats)

    def reconstruct_absolute(self, c2d, c3d, k):
        return self.eng.reconstruct_absolute(c2d, c3d, k)

    def combine_latents(self, points):
        return self.eng.combine_latents(points)

    def allgather(self, padded):
        n = self.crops.shape[0]
        out = torch.zeros((self.world,) + tuple(padded.shape), dtype=padded.dtype, device=padded.device)
        for r in range(self.world):
            s, e = parallel.shard_range(n, self.world, r)
            if r == self.rank:
                out[r] = padded
            elif e > s:
                if (s, e) not in self.decoded:
                    self.decoded[(s, e)] = parallel.pack_decoded(*self.eng.head_decode(self.eng.backbone(self.crops[s:e])))
                out[r, :e - s] = self.decoded[(s, e)]
        return out


def check_sharded(eng, crops, intr, cases, expected, log):
    """ShardedMetrabs.forward on every simulated rank of each (n, W) in cases equals expected[n] (forward on crops[:n])."""
    bad = []
    for n, w in cases:
        decoded = {}
        for r in range(w):
            out = parallel.ShardedMetrabs(None, r, w, engine=SimulatedRanks(eng, crops[:n], r, w, decoded)).forward(
                crops[:n], intr[:n])
            if not torch.equal(out, expected[n]):
                bad.append(f'sharded n={n} W={w} rank {r}: max |diff| {float((out - expected[n]).abs().max()):.3e}')
        log.append(f'{n}/{w}')
    return bad


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('config', list(CONFIGS))
def test_batch_invariance(H, affine_path, config, precision):
    t0 = time.perf_counter()
    m, side = make_model(H, config, precision, affine_path)
    eng = m.engine()
    n = CONFIGS[config][1]
    crops_all, intr_all = (t.cuda() for t in port.synthetic_inputs(n + 1, side, seed=11))
    crops, intr = crops_all[:n], intr_all[:n]

    eng.profile_begin()
    feats = eng.backbone(crops)
    c2d, c3d = eng.head_decode(feats)
    head_cls = set(eng.profile_end())
    joints = eng.forward(crops, intr)
    torch.cuda.synchronize()
    assert all(torch.isfinite(t).all() for t in (feats, c2d, c3d, joints)), 'non-finite anchor results'
    assert c2d.shape == (n, eng.n_points, 2) and c3d.shape == (n, eng.n_points, 3) and joints.shape == (n, eng.n_out, 3)
    fused_head = 'tc_head_softargmax_kernel' in head_cls
    assert fused_head == (precision in T16 and head_cpt(eng.feature_side ** 2) is not None), head_cls

    bad, first_bad = [], []
    checked = []
    prefix_joints = {n: joints}
    moved = 0  # sub-batches whose joints differ from the anchor's rows (batch-global RMS)
    for s, e in sub_batches(n):
        c, k = crops[s:e], intr[s:e]
        f = eng.backbone(c)
        a2, a3 = eng.head_decode(f)
        for nm, x, ref in (('features', f, feats[s:e]), ('coords2d', a2, c2d[s:e]), ('coords3d_rel', a3, c3d[s:e])):
            if not torch.equal(x, ref):
                d = (x.float() - ref.float()).abs().flatten(1).amax(1)
                rows = torch.nonzero(d != 0).flatten().tolist()
                bad.append(f'[{s}, {e}) {nm}: rows {[s + i for i in rows[:16]]} differ (max |diff| {float(d.max()):.3e})')
                first_bad.append((s, e))
        j = eng.forward(c, k)
        rec = eng.combine_latents(eng.reconstruct_absolute(a2, a3, k))
        if not torch.equal(j, rec):
            bad.append(f'[{s}, {e}) joints: forward != reconstruct_absolute of its own decode '
                       f'(max |diff| {float((j - rec).abs().max()):.3e})')
        moved += not torch.equal(j, joints[s:e])
        if s == 0:
            prefix_joints[e] = j
        checked.append(f'{s}:{e}')
    # the anchor plus one crop: its first n rows are the anchor's
    f1 = eng.backbone(crops_all)
    e2, e3 = eng.head_decode(f1)
    for nm, x, ref in (('features', f1[:n], feats), ('coords2d', e2[:n], c2d), ('coords3d_rel', e3[:n], c3d)):
        if not torch.equal(x, ref):
            bad.append(f'[0, {n + 1}) {nm}: the anchor rows differ')
    checked.append(f'0:{n + 1}')
    del f, f1
    if first_bad:
        bad.append('first differing op, ' + first_differing_op(eng, crops, *first_bad[0]))
    assert not bad, f'{config} x{n} [{precision}]:\n  ' + '\n  '.join(bad)
    # sensitivity control: the comparison above can fail - the reconstruction's batch-global RMS moves the joints
    assert moved > 0, 'every sub-batch reproduced the anchor joints: the joint comparison would miss a difference'

    # what the sub-batch sizes reached
    batches = sorted({e - s for s, e in sub_batches(n)} | {n, n + 1})
    reached, seen = tails_reached(eng, precision, batches, fused_head)
    t16, t32 = TAILS[config]
    expected = t16 if precision in T16 else t32 if precision == 'tf32x3' else ({'se'} & t32)
    assert reached == expected, (f'{config} [{precision}]: tails reached {sorted(reached)}, expected {sorted(expected)}; '
                                 f'{seen}')

    # guard bands: the rows behind a prefix view of the output and the workspace bytes past this batch's layout
    for b in (1, 33, n - 1):
        buf = torch.full((b + 5, eng.n_out, 3), float('nan'), device=crops.device)
        eng.forward(crops[:b], intr[:b], out=buf[:b])
        torch.cuda.synchronize()
        assert torch.isnan(buf[b:]).all(), f'forward of {b} crops wrote past its output rows'
        assert torch.equal(buf[:b], prefix_joints[b]), b
    eng.forward(crops_all, intr_all)  # the workspace now holds n + 1 crops
    for b in (1, 33, n - 1):
        ws = eng.workspace(n + 1)
        need = _lib.lib().mtb_workspace_bytes(eng._h, b)
        assert ws.numel() > need
        ws[need:] = 0xA5
        j = eng.forward(crops[:b], intr[:b])
        torch.cuda.synchronize()
        n_bad = sum(int(torch.count_nonzero(c != 0xA5)) for c in ws[need:].split(1 << 28))
        assert n_bad == 0, f'a forward of {b} crops wrote {n_bad} bytes past mtb_workspace_bytes({b}) = {need}'
        assert torch.equal(j, prefix_joints[b]), b

    # ShardedMetrabs.forward with every rank simulated here: equal and ragged shards, fewer crops than ranks
    log = []
    bad = check_sharded(eng, crops, intr, [(n, 2), (n, 4), (n, 8), (n - 1, 8), (3, 4), (3, 8)],
                        {k: prefix_joints[k] for k in (n, n - 1, 3)}, log)
    assert not bad, f'{config} x{n} [{precision}]:\n  ' + '\n  '.join(bad)

    print(f'{config} x{n} [{precision}]: {len(checked)} sub-batches {" ".join(checked)}; sharded (n/W) {" ".join(log)}; '
          f'tails {sorted(reached)} {seen}; head {"fused" if fused_head else "unfused"}; '
          f'{time.perf_counter() - t0:.1f} s')
    del m, eng, feats
    torch.cuda.empty_cache()


@pytest.mark.parametrize('precision', MODES)
@pytest.mark.parametrize('config', ['bench', 'latent'])
def test_forward_sharded_world_one(H, affine_path, config, precision):
    """mtb_forward_sharded on a world-size-1 NCCL communicator (pack, all-gather, unpack, the scratch layout, the latent
    recombination) equals forward bit for bit, directly and through ShardedMetrabs."""
    m, side = make_model(H, config, precision, affine_path)
    eng = m.engine()
    eng.comm_init(0, 1, lambda raw: raw)
    for b in (CONFIGS[config][1], 33, 1):
        crops, intr = (t.cuda() for t in port.synthetic_inputs(b, side, seed=12))
        ref = eng.forward(crops, intr)
        out = eng.forward_sharded(crops, intr)
        out2 = parallel.ShardedMetrabs(m, 0, 1).forward(crops, intr)
        torch.cuda.synchronize()
        assert out.shape == (b, eng.n_out, 3)
        assert torch.equal(out, ref) and torch.equal(out2, ref), (b, float((out - ref).abs().max()))
    del m, eng
    torch.cuda.empty_cache()


@pytest.mark.parametrize('precision', MODES)
def test_pipelined_host_slots(H, affine_path, precision):
    """forward_host_submit / _wait with two different batches (256 and 255 crops) on slots 0 and 1, then the slots reused
    with the batches swapped: every result is forward's on that batch's own crops."""
    m, side = make_model(H, 'bench', precision, affine_path)
    eng = m.engine()
    batches = [port.synthetic_inputs(256, side, seed=13), port.synthetic_inputs(255, side, seed=14)]
    host = [(c.contiguous().pin_memory(), k.contiguous().pin_memory()) for c, k in batches]
    refs = [eng.forward(c.cuda(), k.cuda()).cpu() for c, k in batches]
    for order in ((0, 1), (1, 0), (0, 1)):
        outs = [torch.full((host[i][0].shape[0], eng.n_out, 3), float('nan')).pin_memory() for i in order]
        for slot, i in enumerate(order):
            eng.forward_host_submit(host[i][0], host[i][1], outs[slot], slot)
        for slot in (0, 1):
            eng.forward_host_wait(slot)
        for slot, i in enumerate(order):
            assert torch.equal(outs[slot], refs[i]), (order, slot, float((outs[slot] - refs[i]).abs().nan_to_num(1e30).max()))
    del m, eng
    torch.cuda.empty_cache()
