"""GPU: the host launch path of the TMA kernels.

* Tensor-map reuse and eviction: one handle per tensor-core mode runs more distinct (workspace, batch) keys than a weight
  set's map cache holds (16), then all of them again, so early keys are evicted and re-encoded.  Every output must be
  bit-equal (torch.equal) to that of a fresh handle, whose maps were all encoded for exactly that call.  The plans are
  checked to reach every cached kernel: fmb_kernel, the TMA depthwise kernel and the fused head in the 16-bit modes,
  tc32_conv_kernel for the convs and the head in tf32x3.
* Two devices in one process (skipped with fewer than two): the dynamic shared-memory opt-in of the >48 KB kernels is per
  device, so bf16 handles on cuda:0 and cuda:1 must both run."""
import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu

NAME, SIDE, J = 'efficientnetv2-tiny', 128, 8


@pytest.fixture(scope='module')
def H():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from tests import helpers
    return helpers


def _model(H, sd, precision, device=0):
    return H.device_model(NAME, port.PathConfig(proc_side=SIDE), J, sd, precision=precision).to(torch.device('cuda', device))


def _check_plan(eng, precision, crops, k):
    from metrabs_b200 import _lib
    names = eng.op_names()
    eng.profile_begin()
    eng.forward(crops, k)
    torch.cuda.synchronize()
    classes = eng.profile_end()
    if precision == 'tf32x3':
        tc32_ops = sum(1 for op in eng.profile_op_times() if op[1] == 'tc32_conv_kernel')
        assert tc32_ops > 0, classes
        assert classes['tc32_conv_kernel']['launches'] == tc32_ops + 1, classes  # + the head's 1x1 conv
        assert 'head_conv(conv_igemm_kernel)' not in classes, classes
    else:
        assert any(eng.op_is_fused_block(i) for i in range(len(names)))
        dw = [i - 1 for i, nm in enumerate(names) if nm.endswith('.avgpool')]
        assert any(eng.op_kernel(i) == _lib.DW_TMA for i in dw)
        assert {'fmb_kernel', 'tc_head_softargmax_kernel', 'tc_conv_kernel'} <= set(classes), classes
        assert 'dwconv_kernel' in classes, classes  # the depthwise class, which includes the TMA kernel


@pytest.mark.parametrize('precision', ['bf16', 'fp16', 'tf32x3'])
def test_map_cache_eviction_and_reencoding(H, precision):
    sd = port.make_effnet_state_dict(port.effnet_spec(NAME), port.PathConfig(proc_side=SIDE), J, seed=0, calib_batch=1)
    eng = _model(H, sd, precision).engine()
    batches = list(range(1, 21))  # more (workspace, batch) keys than a cache entry set holds
    inputs = {b: tuple(t.cuda() for t in port.synthetic_inputs(b, SIDE, seed=b)) for b in batches}
    _check_plan(eng, precision, *inputs[3])
    ref = {}
    for b in batches:
        ref[b] = _model(H, sd, precision).engine().forward(*inputs[b])
    for rnd in range(2):
        for b in batches:
            out = eng.forward(*inputs[b])
            assert torch.equal(out, ref[b]), (precision, rnd, b, float((out - ref[b]).abs().max()))


def test_two_devices_in_one_process(H):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 CUDA devices')
    sd = port.make_effnet_state_dict(port.effnet_spec(NAME), port.PathConfig(proc_side=SIDE), J, seed=0, calib_batch=1)
    crops, k = port.synthetic_inputs(3, SIDE, seed=5)
    outs = []
    for dev in (0, 1):
        eng = _model(H, sd, 'bf16', dev).engine(torch.device('cuda', dev))
        out = eng.forward(crops.to(eng.device), k.to(eng.device))
        torch.cuda.synchronize(dev)
        assert torch.isfinite(out).all()
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
