"""GPU: the scheduling corners of the persistent fmb_kernel (one CTA per SM walking 16 x 8 output tiles, the input of a tile
loaded once as three column-shifted boxes and kept across its expanded-channel chunks).  Every case must be bit-equal
(torch.equal) to the two-launch path (two tc_conv_kernel launches with the same MMA order and roundings):

* EfficientNetV2-L@32 stage 2 (an 8 x 8 map: one tile per crop, most of its 16 x 10-pixel boxes outside the map) at 1, 2
  and 3 crops (fewer tiles than SMs), 133 crops (one CTA takes a second tile) and 265 crops (one CTA takes a third);
* EfficientNetV2-L@256 stage 3 (Cin 96: two k-chunks, boxes of both resident) at a tile count just past a multiple of the
  grid, so most CTAs reuse their box buffer for a second tile and a few for a third."""
import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def _engine(H, side, precision):
    name = 'efficientnetv2-l'
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=1)
    return H.device_model(name, pcfg, 8, sd, precision=precision).engine()


def _fused_vs_two_launches(eng, nm, batch, dtype, seed):
    i = eng.op_names().index(nm)
    assert eng.op_is_fused_block(i)
    io = eng.op_io(i)
    x = torch.randn((batch,) + io['in_shape'], generator=torch.Generator().manual_seed(seed)).to(dtype).float().cuda()
    out = eng.debug_run_fused_block(i, x)
    mid = eng.debug_run_op(i, x)
    two = eng.debug_run_op(i + 1, mid, x if eng.op_io(i + 1)['residual'] else None)
    assert torch.isfinite(out).all()
    assert torch.equal(out, two), (nm, batch, float((out - two).abs().max()))
    return io


@pytest.mark.parametrize('precision,dtype', [('bf16', torch.bfloat16), ('fp16', torch.float16)])
def test_fmb_persistent_one_tile_per_crop(H, precision, dtype):
    eng = _engine(H, 32, precision)
    for batch in [1, 2, 3, 133, 265]:
        io = _fused_vs_two_launches(eng, 'backbone.1.2.1.block.0', batch, dtype, batch)
        assert io['in_shape'] == (8, 8, 64), io


def test_fmb_persistent_stage3_tail(H):
    eng = _engine(H, 256, 'bf16')
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles_per_crop = 2 * 4  # a 32 x 32 map in 16 x 8 tiles
    batch = 2 * sms // tiles_per_crop + 1
    tiles = batch * tiles_per_crop
    assert tiles > 2 * sms and tiles % sms != 0, (tiles, sms)
    io = _fused_vs_two_launches(eng, 'backbone.1.3.1.block.0', batch, torch.bfloat16, 7)
    assert io['in_shape'] == (32, 32, 96), io
