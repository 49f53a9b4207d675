"""GPU: the squeeze-excitation (SE) scale of the 16-bit projection GEMMs (bf16, fp16), applied by tc_conv_kernel to its
landed A tiles in shared memory for projections to at most 256 channels, by se_scale_kernel ahead of the wider ones.

* Placement, bit for bit: for every distinct SE projection shape of EfficientNetV2-L@256 at 97 crops (M tails, two crops
  per 128-row tile on 8x8 maps), EfficientNetV2-S@224 (7x7 maps: tiles straddle three crops at irregular offsets),
  EfficientNet-B0@224 (Cin = 144, 672, ...: partial 64-channel k-blocks) and MobileNetV3-Large@256 (hard-sigmoid SE,
  narrow Cin), debug_run_op(x, res, s) must equal debug_run_op(q(q(x) * s), res, 1) with s random per (crop, channel) and q
  the rounding to the mode's type.  A scale of exactly 1.0 leaves the pre-rounded input as it is, so the second call is the
  plain GEMM on what the first must have scaled to: it pins the row -> crop and swizzled chunk -> channel mapping without
  relying on the kernel's own scaling.
* Which projections keep the separate pass: in a profiled EfficientNetV2-L forward only the SE projections to more than
  256 channels launch se_scale_kernel."""
import pytest
import torch

from oracle import port, port_effnet_b, port_mobilenet, port_ops
from oracle import port_tf_backbones as tfb
from tests.test_gpu_ops16_vs_conv2d import op_classes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def engine(H, name, side, precision):
    if name == 'mobilenetv3-large':
        from tests.test_gpu_mobilenet_large import device_model
        pcfg = port.PathConfig(proc_side=side, stride_test=32, depth=8)
        sd = tfb.make_state_dict(port_mobilenet.MobileNetV3Spec(pcfg, 'large'), pcfg, 8, seed=0, calib_batch=1)
        return device_model(H, 'large', pcfg, 8, sd, precision).engine()
    pcfg = port.PathConfig(proc_side=side)
    if name.startswith('efficientnet-b'):
        from tests.test_gpu_effnet_b import device_model
        sd = port_effnet_b.make_state_dict(port_effnet_b.effnet_b_spec(name), pcfg, 8, seed=0, calib_batch=1)
        return device_model(H, name, pcfg, 8, sd, precision).engine()
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0, calib_batch=1)
    return H.device_model(name, pcfg, 8, sd, precision=precision).engine()


CASES = [('efficientnetv2-l', 256, 97), ('efficientnetv2-s', 224, 5), ('efficientnet-b0', 224, 3),
         ('mobilenetv3-large', 256, 3)]


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
@pytest.mark.parametrize('name,side,batch', CASES)
def test_se_scale_placement_is_bit_exact(H, precision, name, side, batch):
    eng = engine(H, name, side, precision)
    classes = op_classes(eng, side)
    st = port_ops.MODES[precision][0]
    q = lambda t: t.to(st).float()  # noqa: E731
    g = torch.Generator().manual_seed(side + batch)
    seen, reached = set(), set()
    for i, nm in enumerate(eng.op_names()):
        io = eng.op_io(i)
        if not io['scale']:
            continue
        sig = (io['in_shape'], io['out_shape'], io['residual'])
        if sig in seen:
            continue
        seen.add(sig)
        assert classes[nm] == 'tc_conv_kernel', (nm, classes[nm])
        (hh, ww, cin), out_shape = io['in_shape'], io['out_shape']
        x = q(3 * torch.randn((batch, hh, ww, cin), generator=g))
        s = 2 * torch.rand(batch, cin, generator=g)
        res = q(torch.randn((batch,) + out_shape, generator=g)).cuda() if io['residual'] else None
        scaled = q(x * s[:, None, None, :])
        x, s, scaled = x.cuda(), s.cuda(), scaled.cuda()
        a = eng.debug_run_op(i, x, res, s)
        b = eng.debug_run_op(i, scaled, res, torch.ones_like(s))
        assert torch.isfinite(a).all(), nm
        assert torch.equal(a, b), (nm, precision, int((a != b).sum()), a.numel())
        rows = batch * hh * ww
        reached |= {('M tail', rows % 128 != 0), ('two crops per tile', hh * ww <= 64),
                    ('three crops per tile', hh * ww < 64), ('partial k-block', cin % 64 != 0),
                    ('residual', io['residual'])}
    print(f'{name}@{side} x{batch} [{precision}]: {len(seen)} SE projection shapes bit-exact')
    assert seen
    if name == 'efficientnetv2-l':
        assert {('M tail', True), ('two crops per tile', True), ('residual', True)} <= reached, reached
    if name == 'efficientnetv2-s':
        assert ('three crops per tile', True) in reached, reached
    if name == 'efficientnet-b0':
        assert ('partial k-block', True) in reached, reached


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_separate_se_pass_only_behind_wide_projections(H, precision):
    """tc_se_in_gemm: projections to at most 256 channels (two N tiles) scale their A tiles themselves, the wider ones run
    behind se_scale_kernel.  EfficientNetV2-L: 10 + 19 SE projections to 192 / 224 channels, 25 + 7 to 384 / 640."""
    eng = engine(H, 'efficientnetv2-l', 256, precision)
    names = eng.op_names()
    se_ops = {nm: eng.op_io(i)['out_shape'][2] for i, nm in enumerate(names) if eng.op_io(i)['scale']}
    assert len(se_ops) == 61
    eng.profile_begin()
    eng.backbone(port.synthetic_inputs(2, 256, seed=3)[0].cuda())
    prof = eng.profile_end()
    per_op = {nm: cls for nm, cls, *_ in eng.profile_op_times()}
    assert all(per_op[nm] == 'tc_conv_kernel' for nm in se_ops)
    wide = sum(c > 256 for c in se_ops.values())
    assert wide == 32
    assert prof['se_scale_kernel']['launches'] == wide, prof['se_scale_kernel']
