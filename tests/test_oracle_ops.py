"""CPU: the per-layer reference (oracle/port_ops.py) reproduces the layer taps of the pinned whole-path port
(oracle/port.py, itself checked against the unmodified reference's goldens in test_oracle_golden.py)."""
import torch

from oracle import port, port_ops


def test_layer_reference_matches_port_taps():
    pcfg = port.PathConfig(proc_side=64)
    spec = port.effnet_spec('efficientnetv2-tiny')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0)
    crops, _ = port.synthetic_inputs(2, 64, seed=0)
    tap = {}
    with torch.inference_mode():
        port.effnet_features(sd, spec, crops, tap=tap)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
    P = 'backbone.1'
    cases = [
        (f'{P}.0', crops, None, tap[f'{P}.0']),                                        # stem (NCHW crops in)
        (f'{P}.1.0.block.0', nhwc(tap[f'{P}.0']), nhwc(tap[f'{P}.0']), tap[f'{P}.1.0']),  # expand-1 fused block + residual
        (f'{P}.2.0.block.0', nhwc(tap[f'{P}.1.0']), None, tap[f'{P}.2.0.block.0']),    # 3x3 stride 2
        (f'{P}.2.1.block.1', nhwc(tap[f'{P}.2.1.block.0']), nhwc(tap[f'{P}.2.0']), tap[f'{P}.2.1']),  # project + residual
        (f'{P}.4.0.block.0', nhwc(tap[f'{P}.3.0']), None, tap[f'{P}.4.0.block.0']),    # MBConv expand
        (f'{P}.4.0.block.1', nhwc(tap[f'{P}.4.0.block.0']), None, tap[f'{P}.4.0.block.1']),  # depthwise stride 2
        (f'{P}.7', nhwc(tap[f'{P}.6.1']), None, tap[f'{P}.7']),                        # last conv
    ]
    for name, x, res, want in cases:
        got = port_ops.conv_layer_reference(sd, spec, name, x, res, dtype=torch.float64).permute(0, 3, 1, 2)
        assert port.relative_error(got, want) < 2e-6, name
    # squeeze-excitation projection: scale * x then 1x1 conv (efficientnet.py:110-173)
    key = f'{P}.4.0.block'
    dw = tap[f'{key}.1']
    s = dw.mean(dim=(2, 3), keepdim=True)
    s = torch.nn.functional.silu(torch.nn.functional.conv2d(s, sd[f'{key}.2.fc1.weight'], sd[f'{key}.2.fc1.bias']))
    s = torch.sigmoid(torch.nn.functional.conv2d(s, sd[f'{key}.2.fc2.weight'], sd[f'{key}.2.fc2.bias']))
    got = port_ops.conv_layer_reference(sd, spec, f'{key}.3', nhwc(dw), None, scale=s[:, :, 0, 0], dtype=torch.float64)
    assert port.relative_error(got.permute(0, 3, 1, 2), tap[f'{key}.3']) < 2e-6


def test_bf16_rounding_points():
    """'bf16' precision rounds the folded weight once and the (scaled) input once; everything else stays wide."""
    pcfg = port.PathConfig(proc_side=64)
    spec = port.effnet_spec('efficientnetv2-tiny')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0)
    x = torch.randn(2, 16, 16, 16).bfloat16().float()
    a = port_ops.conv_layer_reference(sd, spec, 'backbone.1.3.0.block.0', x, precision='bf16')
    b = port_ops.conv_layer_reference(sd, spec, 'backbone.1.3.0.block.0', x, precision='exact')
    err = port.relative_error(a, b)
    assert 1e-5 < err < 2e-2  # differs by the weight rounding only


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def test_tf_backbone_op_tables_match_port_taps():
    """resnet50_op_table / mobilenetv3_small_op_table restate the layers of port_tf_backbones: caffe / 2x-1 stems, the
    zero-padded max pool, dense-SAME strided 1x1 sampled at shift::stride, dilated 3x3, relu(shortcut + _3_conv),
    correct_pad, hard-swish, SE (ReLU / hard-sigmoid) scaled projection + residual, Conv_2 with bias."""
    from oracle import port_tf_backbones as tfb
    P = 'backbone.'
    for stride, centered in [(8, True), (32, True), (16, False)]:
        pcfg = port.PathConfig(proc_side=64, stride_test=stride, centered_stride=centered)
        spec = tfb.ResNet50Spec(pcfg)
        sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
        crops, _ = port.synthetic_inputs(2, 64, seed=1)
        tap = {}
        with torch.inference_mode():
            spec.features(sd, crops, tap=tap)
        table = port_ops.resnet50_op_table(pcfg)
        cases = [('conv1_conv', crops, None), ('pool1_pool', _nhwc(tap[P + 'conv1_conv']), None)]
        prev = P + 'pool1_pool'
        for name, _f, st, shift, dil, conv_shortcut in tfb.resnet50_blocks(pcfg):
            if conv_shortcut or dil > 1:
                if conv_shortcut:
                    cases.append((name + '_0_conv', _nhwc(tap[prev]), None))
                cases.append((name + '_1_conv', _nhwc(tap[prev]), None))
                cases.append((name + '_2_conv', _nhwc(tap[P + name + '_1_conv']), None))
            if not conv_shortcut:  # identity shortcut: relu(block input + _3_conv)
                cases.append((name + '_3_conv', _nhwc(tap[P + name + '_2_conv']), _nhwc(tap[prev])))
            prev = P + name + '_3_conv'
        seen = set()
        for name, x, res in cases:
            op = table[P + name]
            seen |= {('shift', op.get('shift', 0)), ('dil', op.get('dil', 1)), ('res_first', op.get('res_first', False))}
            got = port_ops.conv_layer_reference(sd, spec, P + name, x, res).permute(0, 3, 1, 2)
            # the _3_conv of an identity block is tapped after the residual; the port evaluates in fp32
            assert port.relative_error(got, tap[P + name]) < 2e-6, (stride, name)
        assert ('res_first', True) in seen
        assert ('shift', 1) in seen or not centered
        assert ('dil', 2) in seen or stride == 32

    pcfg = port.PathConfig(proc_side=64, stride_test=32)
    spec = tfb.MobileNetV3SmallSpec(pcfg)
    sd = tfb.make_state_dict(spec, pcfg, 8, seed=0, calib_batch=2)
    crops, _ = port.synthetic_inputs(2, 64, seed=1)
    tap = {}
    with torch.inference_mode():
        spec.features(sd, crops, tap=tap)
    b = P + 'expanded_conv_4'
    dw = tap[b + '.depthwise']
    q = torch.nn.functional.relu(torch.nn.functional.conv2d(dw.mean(dim=(2, 3), keepdim=True), sd[b + '.squeeze_excite.Conv.weight'],
                                                            sd[b + '.squeeze_excite.Conv.bias']))
    q = tfb.hard_sigmoid(torch.nn.functional.conv2d(q, sd[b + '.squeeze_excite.Conv_1.weight'], sd[b + '.squeeze_excite.Conv_1.bias']))
    cases = [('Conv', crops, None, None), ('expanded_conv.depthwise', _nhwc(tap[P + 'Conv']), None, None),
             ('expanded_conv_1.expand', _nhwc(tap[P + 'expanded_conv.project']), None, None),
             ('expanded_conv_3.depthwise', _nhwc(tap[P + 'expanded_conv_3.expand']), None, None),
             ('expanded_conv_8.depthwise', _nhwc(tap[P + 'expanded_conv_8.expand']), None, None),  # bottom-right stride 2
             ('expanded_conv_4.project', _nhwc(dw), _nhwc(tap[P + 'expanded_conv_3.project']), q[:, :, 0, 0]),
             ('Conv_1', _nhwc(tap[P + 'expanded_conv_10.project']), None, None), ('Conv_2', _nhwc(tap[P + 'Conv_1']), None, None)]
    for name, x, res, s in cases:
        got = port_ops.conv_layer_reference(sd, spec, P + name, x, res, s).permute(0, 3, 1, 2)
        assert port.relative_error(got, tap[P + name]) < 2e-6, name
    assert port_ops.mobilenetv3_small_op_table(pcfg)[P + 'expanded_conv_8.depthwise']['shift'] == 1


# ---- the per-element bound (port_ops.layer_bound / check_bound), checked against emulated device results --------------
def _round_sig(t, bits):
    """t rounded to ``bits`` significant bits (the result of an approximation with ~2^-bits relative error)."""
    m, e = torch.frexp(t)
    return torch.ldexp(torch.round(m * 2.0 ** bits) / 2.0 ** bits, e)


def _tiny():
    pcfg = port.PathConfig(proc_side=64)
    spec = port.effnet_spec('efficientnetv2-tiny')
    return spec, port.make_effnet_state_dict(spec, pcfg, 8, seed=0)


def _operands(shape_x, shape_res, cin, st, seed, scale=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape_x, generator=g).to(st).double()
    res = torch.randn(shape_res, generator=g).to(st).double() if shape_res is not None else None
    s = torch.rand(shape_x[0], cin, generator=g).float() if scale else None
    return x, res, s


def _emulate(sd, spec, name, x, res, s, precision, act=None, res_first=None):
    """A device result: the layer at ``precision``'s rounding points with a given activation form, rounded once."""
    op = port_ops.op_table(spec)[name]
    y, z, _k = port_ops._layer(sd, spec, name, x, None if res_first is not None else res, s, precision, torch.float64)
    if act is not None or res_first is not None:
        if res_first:
            z = z + res.permute(0, 3, 1, 2)
        y = (act or port_ops._act)(z, op['act']) if act is None else act(z)
        if res_first is False:
            y = y + res.permute(0, 3, 1, 2)
    return _nhwc(y).to(port_ops.MODES[precision][0])


def _silu_tanh_form(z):  # tc_act / fast_act for bf16 outputs, tanh.approx modelled with ~2^-12 relative error
    h = 0.5 * z
    return h + h * _round_sig(torch.tanh(h), 12)


def test_bound_accepts_correctly_rounded_results():
    spec, sd = _tiny()
    table = port_ops.effnet_op_table(spec)
    for precision in port_ops.MODES:
        st = port_ops.MODES[precision][0]
        for name in ['backbone.1.1.0.block.0', 'backbone.1.2.0.block.0', 'backbone.1.4.1.block.1', 'backbone.1.4.1.block.3',
                     'backbone.1.6.0.block.1']:
            w = sd[name + '.0.weight']
            op = table[name]
            h = 16 if op['stride'] == 1 else 32
            cin = w.shape[0] if op['depthwise'] else w.shape[1]
            has_res = name.endswith('.3') or name == 'backbone.1.1.0.block.0'
            hout = h // op['stride']
            x, res, s = _operands((2, h, h, cin), (2, hout, hout, w.shape[0]) if has_res else None, cin, st, 1,
                                  scale=name.endswith('.3'))
            ref, tol = port_ops.layer_bound(sd, spec, name, x, res, s, precision)
            # rounded exact result, and an fp32 evaluation (other summation order, fp32 activation) rounded once
            for dev in [ref.to(st), port_ops.conv_layer_reference(sd, spec, name, x.float(), None if res is None else res.float(), s,
                                                                    precision, dtype=torch.float32).to(st)]:
                worst, bad = port_ops.check_bound(dev, ref, tol, precision)
                assert bad == 0, (precision, name, worst)
                assert worst <= 1.0
    # the bf16 tensor-core SiLU (tanh.approx form) is within the bf16-mode bound
    name = 'backbone.1.4.1.block.1'
    x, _r, _s = _operands((2, 16, 16, 128), None, 128, torch.bfloat16, 2)
    ref, tol = port_ops.layer_bound(sd, spec, name, x, None, None, 'bf16')
    assert port_ops.check_bound(_emulate(sd, spec, name, x, None, None, 'bf16', act=_silu_tanh_form), ref, tol, 'bf16')[1] == 0


def test_bound_rejects_bf16_silu_form_in_fp16():
    """The fp16 kernels' reason for silu_f16out: h + h*tanh.approx(h) stored as fp16 is off by ~2^-11 relative to h^2."""
    spec, sd = _tiny()
    for name, shape in [('backbone.1.4.1.block.1', (2, 16, 16, 128)), ('backbone.1.4.1.block.0', (2, 16, 16, 32))]:
        x, _r, _s = _operands(shape, None, shape[-1], torch.float16, 3)
        ref, tol = port_ops.layer_bound(sd, spec, name, x, None, None, 'fp16')
        worst, bad = port_ops.check_bound(_emulate(sd, spec, name, x, None, None, 'fp16', act=_silu_tanh_form), ref, tol, 'fp16')
        assert bad > 0 and worst > 2, (name, worst)


def test_bound_rejects_one_dropped_border_tap():
    """Output column W-2 computed without tap (1, 2), the one that reads the last input column (a clipped edge)."""
    spec, sd = _tiny()
    for precision in port_ops.MODES:
        st = port_ops.MODES[precision][0]
        for name, cin in [('backbone.1.4.1.block.1', 128), ('backbone.1.2.1.block.0', 16)]:
            x, _r, _s = _operands((2, 8, 8, cin), None, cin, st, 4)
            ref, tol = port_ops.layer_bound(sd, spec, name, x, None, None, precision)
            sd2 = dict(sd)
            sd2[name + '.0.weight'] = sd[name + '.0.weight'].clone()
            sd2[name + '.0.weight'][:, :, 1, 2] = 0
            dev = ref.to(st).clone()
            dev[:, :, -2] = _emulate(sd2, spec, name, x, None, None, precision)[:, :, -2]
            worst, bad = port_ops.check_bound(dev, ref, tol, precision)
            assert bad > 0 and worst > 2, (precision, name, worst)


def test_bound_rejects_residual_before_activation():
    """EfficientNet adds the residual after SiLU; relu(res + x) order (ResNet's) on an EfficientNet op must fail, and the
    EfficientNet order on a ResNet _3_conv must fail."""
    from oracle import port_tf_backbones as tfb
    spec, sd = _tiny()
    name = 'backbone.1.1.0.block.0'
    for precision in port_ops.MODES:
        st = port_ops.MODES[precision][0]
        x, res, _s = _operands((2, 32, 32, 8), (2, 32, 32, 8), 8, st, 5)
        ref, tol = port_ops.layer_bound(sd, spec, name, x, res, None, precision)
        worst, bad = port_ops.check_bound(_emulate(sd, spec, name, x, res, None, precision, res_first=True), ref, tol, precision)
        assert bad > 0 and worst > 2, (precision, worst)
    pcfg = port.PathConfig(proc_side=64, stride_test=32)
    rspec = tfb.ResNet50Spec(pcfg)
    rsd = tfb.make_state_dict(rspec, pcfg, 8, seed=0, calib_batch=1)
    name = 'backbone.conv2_block2_3_conv'
    for precision in port_ops.MODES:
        st = port_ops.MODES[precision][0]
        x, res, _s = _operands((2, 16, 16, 64), (2, 16, 16, 256), 64, st, 6)
        ref, tol = port_ops.layer_bound(rsd, rspec, name, x, res, None, precision)
        assert port_ops.check_bound(ref.to(st), ref, tol, precision)[1] == 0
        worst, bad = port_ops.check_bound(_emulate(rsd, rspec, name, x, res, None, precision, res_first=False), ref, tol, precision)
        assert bad > 0 and worst > 2, (precision, worst)


def test_bound_rejects_unrounded_se_scale_in_tensor_core_modes():
    """se_scale_kernel rounds x*s to 16 bits ahead of the tensor-core GEMM; a device that kept the fp32 product (what the
    CUDA-core modes do) fails the tensor-core bound, and the CUDA-core bound rejects the rounded product."""
    spec, sd = _tiny()
    name = 'backbone.1.4.1.block.3'  # 128 -> 32 projection with SE scale
    for tc, simt in [('bf16', 'bf16_simt'), ('fp16', 'fp16_simt')]:
        st = port_ops.MODES[tc][0]
        x, res, s = _operands((4, 16, 16, 128), (4, 16, 16, 32), 128, st, 7, scale=True)
        for want, other in [(tc, simt), (simt, tc)]:
            ref, tol = port_ops.layer_bound(sd, spec, name, x, res, s, want)
            assert port_ops.check_bound(_emulate(sd, spec, name, x, res, s, want), ref, tol, want)[1] == 0
            worst, bad = port_ops.check_bound(_emulate(sd, spec, name, x, res, s, other), ref, tol, want)
            assert bad > 0 and worst > 1.5, (want, worst)


def test_bound_fp16_overflow():
    """Overflow gives inf, no saturation: inf is required where the result surely overflows, allowed only within the
    bound of the threshold, and a finite value there (saturation) fails."""
    spec, sd = _tiny()
    name = 'backbone.1.4.1.block.0'
    x, _r, _s = _operands((2, 8, 8, 32), None, 32, torch.float16, 8)
    x = (x * 20000).clamp(-60000, 60000).half().double()
    ref, tol = port_ops.layer_bound(sd, spec, name, x, None, None, 'fp16')
    dev = ref.half()
    assert torch.isinf(dev).any() and torch.isfinite(dev).any()
    assert port_ops.check_bound(dev, ref, tol, 'fp16')[1] == 0
    sat = dev.clone()
    sat[torch.isinf(sat)] = torch.sign(sat[torch.isinf(sat)]) * 65504
    assert port_ops.check_bound(sat, ref, tol, 'fp16')[1] > 0
    nan = dev.clone()
    nan.view(-1)[0] = float('nan')
    assert port_ops.check_bound(nan, ref, tol, 'fp16')[1] == 1
