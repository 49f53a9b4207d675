"""GPU: the fused FusedMBConv kernel (fmb_kernel, csrc/tc_fmb.cuh: 3x3 expand + SiLU -> 1x1 projection + residual in ONE
launch, the expanded tile never leaves the SM) against

* plain ``torch.nn.functional.conv2d`` arithmetic (oracle/port_ops.py restates the two reference layers,
  metrabs_pytorch/backbones/efficientnet.py:176-234 of the reference) on the same bf16-rounded input and weights, with the
  expanded activation rounded to bf16 between the two convs (what the unfused path stores): bar = one bf16 ulp of the
  output plus the propagated ulp flips of the intermediate (1e-2 on ||.||inf/||ref||inf; a descriptor / layout / pipeline
  bug gives O(1) errors);
* the unfused device path (two tc_conv_kernel launches) on identical inputs: same MMA order and roundings, so equal up to
  one bf16 ulp;
* in bf16 and fp16, element by element: the unfused path's 16-bit intermediate within port_ops.layer_bound of the expand
  conv, and the fused output within the bound of the projection evaluated on that intermediate.  This assumes the fused
  kernel's own intermediate is bit-equal to the unfused one (same MMA order, bias, activation and rounding); the test
  asserts it where it can, by requiring the fused output to be bit-equal to the two-launch output."""
import pytest
import torch

from oracle import port, port_ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from tests import helpers
    return helpers


def _block_reference(sd, spec, names, i, x, precision='bf16'):
    """expand conv -> 16 bits -> projection (+ residual x) with conv2d, fp32 accumulate on the GPU."""
    y = port_ops.conv_layer_reference(sd, spec, names[i], x, precision=precision, dtype=torch.float32)
    y = y.to(port_ops.MODES[precision][0]).float()
    return port_ops.conv_layer_reference(sd, spec, names[i + 1], y, x, precision=precision, dtype=torch.float32)


def _check_elementwise(sd, spec, names, i, x, res, mid, out, precision):
    """-> worst |dev-ref|/tol of the intermediate and of the fused output (on the device's own intermediate)."""
    worst = []
    for nm, xin, res, dev in [(names[i], x, None, mid), (names[i + 1], mid, res, out)]:
        ref, tol = port_ops.layer_bound(sd, spec, nm, xin.double(), None if res is None else res.double(), None, precision)
        w, bad = port_ops.check_bound(dev, ref, tol, precision)
        assert bad == 0, (nm, precision, bad, w)
        worst.append(w)
    return worst


@pytest.mark.parametrize('name,side,batch', [('efficientnetv2-s', 256, 3), ('efficientnetv2-l', 256, 2), ('efficientnetv2-l', 384, 1),
                                             ('efficientnetv2-m', 192, 2), ('efficientnetv2-tiny', 64, 5),  # tiny: Cin 16, one 64-wide chunk
                                             ('efficientnetv2-l', 32, 3)])  # 8x8 / 4x4 maps, 3 crops: tiles mostly outside the map
@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_fused_block_vs_conv2d_and_unfused(H, name, side, batch, precision):
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    st = port_ops.MODES[precision][0]
    eng = H.device_model(name, pcfg, 8, sd, precision=precision).engine()
    names = eng.op_names()
    g = torch.Generator().manual_seed(5)
    seen = set()
    for i, nm in enumerate(names):
        if not eng.op_is_fused_block(i):
            continue
        io = eng.op_io(i)
        if io['in_shape'] in seen:
            continue
        seen.add(io['in_shape'])
        x = torch.randn((batch,) + io['in_shape'], generator=g).to(st).float().cuda()
        out = eng.debug_run_fused_block(i, x)
        ref = _block_reference(sd, spec, names, i, x, precision)
        err = port.relative_error(out.cpu(), ref.cpu())
        mid = eng.debug_run_op(i, x)
        res = x if eng.op_io(i + 1)['residual'] else None
        two = eng.debug_run_op(i + 1, mid, res)
        d = (out - two).abs()
        ulp = two.abs() * 2.0 ** -7 + 2.0 ** -9
        assert bool((d == 0).all()), (nm, float(d.max()))  # the intermediate the bound below is evaluated on
        w_mid, w_out = _check_elementwise(sd, spec, names, i, x, res, mid, out, precision)
        print(f'{name}@{side} {nm} {io["in_shape"]} [{precision}]: fused vs conv2d {err:.2e}; vs unfused device path: '
              f'{float((d == 0).float().mean()) * 100:.2f} % bit-equal, max diff {float(d.max()):.3e}; '
              f'worst |dev-ref|/tol {w_mid:.3g} (expand), {w_out:.3g} (fused output)')
        assert err < 1e-2, (nm, err)
        assert bool((d <= ulp).all()), (nm, float(d.max()))
    assert seen, 'no fused FusedMBConv block in this model'


@pytest.mark.parametrize('batch', [64, 256])
def test_fused_block_at_bench_batch(H, batch):
    """many waves of tiles (8192 / 2048 tiles) on the two EfficientNetV2-L@256 block shapes"""
    name, side = 'efficientnetv2-l', 256
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    eng = H.device_model(name, pcfg, 8, sd, precision='bf16').engine()
    names = eng.op_names()
    g = torch.Generator().manual_seed(6)
    for nm in ['backbone.1.2.1.block.0', 'backbone.1.3.1.block.0']:
        i = names.index(nm)
        assert eng.op_is_fused_block(i)
        x = torch.randn((batch,) + eng.op_io(i)['in_shape'], generator=g).bfloat16().float().cuda()
        out = eng.debug_run_fused_block(i, x)
        ref = _block_reference(sd, spec, names, i, x)
        err = port.relative_error(out.cpu(), ref.cpu())
        print(f'{nm} batch {batch}: fused vs conv2d {err:.2e}')
        assert err < 1e-2, (nm, err)
        del out, ref, x
        torch.cuda.empty_cache()


def test_whole_backbone_with_and_without_fusion(H, monkeypatch):
    """EfficientNetV2-S features through the fused blocks (the unfused op chain via debug_run_op is covered above);
    here: the full forward stays finite and close to the bf16 CUDA-core chain."""
    name, side, batch = 'efficientnetv2-s', 256, 4
    pcfg = port.PathConfig(proc_side=side)
    sd = port.make_effnet_state_dict(port.effnet_spec(name), pcfg, 8, seed=0)
    crops, _ = port.synthetic_inputs(batch, side, seed=0)
    e_tc = H.device_model(name, pcfg, 8, sd, precision='bf16').engine()
    e_ref = H.device_model(name, pcfg, 8, sd, precision='bf16_simt').engine()
    names = e_tc.op_names()
    last_fused = max(i for i in range(len(names)) if e_tc.op_is_fused_block(i))
    a = e_tc.debug_run_ops(crops.cuda(), last_fused + 2)   # through the last fused block
    b = e_ref.debug_run_ops(crops.cuda(), last_fused + 2)
    err = port.relative_error(a.cpu(), b.cpu())
    print(f'{name}: activations after the last fused block vs the CUDA-core bf16 chain: {err:.2e}')
    assert torch.isfinite(a).all() and err < 0.1
