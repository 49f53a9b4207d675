"""CPU: the fp16-storage restatement (oracle/port_f16.py) against the fp32 port and against the bf16-storage restatement on
the conditioned random weights the parity tests use (no kernel of this repo involved).  fp16 keeps 3 more significand
bits than bf16, so storing the activations in fp16 - the arithmetic of the reference's fp16 autocast - must bring the
features several times closer to fp32, without coming near the fp16 range limit (65504) on these fixtures."""
import pytest
import torch

from oracle import port, port_bf16, port_f16


@pytest.mark.parametrize('name,side,j,batch', [('efficientnetv2-tiny', 64, 8, 3), ('efficientnetv2-s', 256, 24, 2),
                                               ('efficientnetv2-l', 256, 24, 2)])
def test_fp16_storage_is_closer_to_fp32_than_bf16(name, side, j, batch):
    pcfg = port.PathConfig(proc_side=side)
    spec = port.effnet_spec(name)
    sd = port.make_effnet_state_dict(spec, pcfg, j, seed=0, calib_batch=2)
    crops, k = port.synthetic_inputs(batch, side, seed=0)
    with torch.inference_mode():
        s_ref, s_b, s_h = {}, {}, {}
        ref = port.metrabs_forward(sd, spec, pcfg, j, crops, k, stages=s_ref)
        out_b = port_bf16.metrabs_forward_bf16(sd, spec, pcfg, j, crops, k, stages=s_b)
        out_h = port_f16.metrabs_forward_f16(sd, spec, pcfg, j, crops, k, stages=s_h)
    e_feat_b = port.relative_error(s_b['features'], s_ref['features'])
    e_feat_h = port.relative_error(s_h['features'], s_ref['features'])
    print(f'{name}@{side}: features bf16 {e_feat_b:.2e} fp16 {e_feat_h:.2e}; joints bf16 '
          f'{port.relative_error(out_b, ref):.2e} fp16 {port.relative_error(out_h, ref):.2e}; max |value| rounded to fp16 '
          f'{s_h["max_abs"]:.1f}')
    assert torch.isfinite(out_h).all()
    assert e_feat_h < 0.25 * e_feat_b
    assert s_h['max_abs'] < 1e3


def test_fp16_restatement_leaves_the_bf16_module_alone():
    """port_f16 runs a private instance of port_bf16: the shared module keeps its bf16 rounding."""
    x = torch.tensor([1.0 + 2.0 ** -9])
    assert float(port_bf16._q(x)) == 1.0             # 8 significand bits: rounds away
    assert float(port_f16._q(x)) == 1.0 + 2.0 ** -9   # 11 significand bits: kept
    assert float(port_f16._q(torch.tensor([1e5]))) == float('inf')  # overflow gives inf, as under autocast
