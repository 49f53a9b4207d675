"""GPU, >= 2 devices (skipped otherwise): the data-parallel path over NCCL - mtb_forward_sharded (local backbone + head
decode, ONE ncclAllGather of [coords2d|coords3d_rel], full-batch reconstruction) must reproduce the UNSHARDED forward of
the concatenated batch on every rank (SURVEY.md 8e; batch-global RMS, ptu3d.py:71-74), including ragged and empty shards.
Every per-crop stage is batch-invariant (test_gpu_batch_invariance.py), so every rank's result equals the unsharded one
bit for bit."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# (model, crop side, joints, crops per rank of the equal-shard case): the small model, and EfficientNetV2-L@256 at c3's
# 32 crops per GPU
MODELS = {'tiny': ('efficientnetv2-tiny', 64, 8, 4), 'l': ('efficientnetv2-l', 256, 24, 32)}


def _worker(rank, world, port_no, precision, model, out_dir):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port_no)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from metrabs_b200 import parallel
    from oracle import port
    from tests import helpers
    name, side, nj, per_rank = MODELS[model]
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, nj, seed=0, **({'calib_batch': 1} if model == 'l' else {}))
    m = helpers.device_model(name, pcfg, nj, sd, precision=precision).to(dev)
    eng = m.engine(dev)

    def bcast(raw):
        t = torch.tensor(list(raw) if raw is not None else [0] * 128, dtype=torch.uint8, device=dev)
        dist.broadcast(t, 0)
        return bytes(t.cpu().tolist())
    eng.comm_init(rank, world, bcast)
    sh = parallel.ShardedMetrabs(m, rank, world)
    res = {}
    for n_total in (world * per_rank, 5, 1):  # equal shards (library path), ragged, fewer crops than ranks
        crops, k = port.synthetic_inputs(n_total, side, seed=3)
        crops, k = crops.to(dev), k.to(dev)
        out = sh.forward(crops, k)
        ref = eng.forward(crops, k)
        torch.cuda.synchronize()
        res[n_total] = (out.cpu(), ref.cpu())
    torch.save(res, os.path.join(out_dir, f'r{rank}.pt'))
    dist.destroy_process_group()


def _run(tmp_path, precision, model, port_no):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 CUDA devices')
    world = 2
    mp.spawn(_worker, args=(world, port_no, precision, model, str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f'r{r}.pt') for r in range(world)]
    _, _, nj, per_rank = MODELS[model]
    for n_total in (world * per_rank, 5, 1):
        for r in range(world):
            out, ref = outs[r][n_total]
            assert out.shape == (n_total, nj, 3)
            assert torch.equal(out, ref), (n_total, r, float((out - ref).abs().max()))
        assert torch.equal(outs[0][n_total][0], outs[1][n_total][0])  # every rank holds the same full result


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_sharded_equals_unsharded_nccl(tmp_path, precision):
    _run(tmp_path, precision, 'tiny', 33500 + (os.getpid() % 2000) + (0 if precision == 'fp32' else 1))


def test_sharded_effnetv2_l_c3_share_nccl(tmp_path):
    """EfficientNetV2-L@256 in bf16 at 2 x 32 crops: c3's share per GPU on the benchmark's model"""
    _run(tmp_path, 'bf16', 'l', 33500 + (os.getpid() % 2000) + 2)
