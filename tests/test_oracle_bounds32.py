"""CPU: the per-element bounds of the fp32-storage modes ('fp32', 'tf32x3') and the per-coordinate bound of the
soft-argmax decode (oracle/port_ops.py), pinned without a GPU.

* 3xTF32: an fp64 emulation of tc32_conv_kernel's split (split_tf32's bit operations in torch, the lo operands truncated
  to tf32 as the tensor core reads them, the lo*lo product dropped) stays within TC32_SPLIT per product and per dot
  product; dropping one of the two correction products exceeds it by orders of magnitude.
* layer_bound in the fp32 modes holds for fp32 evaluations of the layer and rejects a wrong activation.
* pool_mean_bound holds for an fp32 strided-then-tree sum.
* decode_bound holds for logits perturbed by up to delta in the worst direction and rejects a decode that weights one
  column with x + 1."""
import torch
import torch.nn.functional as F

from oracle import port, port_ops


def _tf32_rn(x):
    """split_tf32's hi: (bits + 0x1000) & 0xffffe000 (round to nearest, ties away) on fp32 x."""
    u = x.float().view(torch.int32)
    return ((u + 0x1000) & ~0x1fff).view(torch.float32)


def _tf32_trunc(x):
    """the tensor core's read of an fp32 operand as tf32: the low 13 mantissa bits dropped."""
    return (x.float().view(torch.int32) & ~0x1fff).view(torch.float32)


def _split(x):
    hi = _tf32_rn(x)
    return hi, x.float() - hi  # exact in fp32


def _operands(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    # mantissas over the whole fp32 range of bits, magnitudes over a few binades, both signs
    x = (torch.randn(n, k, generator=g) * torch.exp2(torch.randint(-6, 6, (n, k), generator=g).float())).float()
    w = (torch.randn(k, generator=g) * torch.exp2(torch.randint(-6, 6, (k,), generator=g).float())).float()
    return x, w


def _emulate_3xtf32(x, w, drop=None):
    """fp64 sum of the three products tc32_conv_kernel issues (each exact in fp64: 11 x 11 significant bits)."""
    xh, xl = _split(x)
    wh, wl = _split(w)
    xl, wl = _tf32_trunc(xl), _tf32_trunc(wl)
    terms = {'hh': xh.double() * wh.double(), 'lh': xl.double() * wh.double(), 'hl': xh.double() * wl.double()}
    return sum(t for key, t in terms.items() if key != drop)


def test_tf32_split_is_exact_and_hi_rounds_to_nearest():
    x, _ = _operands(64, 256, seed=1)
    hi, lo = _split(x)
    assert torch.equal(hi.double() + lo.double(), x.double())  # lo = x - hi is exact
    assert bool(((hi.view(torch.int32) & 0x1fff) == 0).all())
    assert bool((lo.double().abs() <= 2.0 ** -11 * x.double().abs()).all())


def test_3xtf32_products_within_the_split_term():
    x, w = _operands(256, 512, seed=2)
    exact = x.double() * w.double()
    mag = (x.double() * w.double()).abs()
    err = (_emulate_3xtf32(x, w) - exact).abs()
    ratio = float((err / (port_ops.TC32_SPLIT * mag)).max())
    assert ratio <= 1.0, ratio
    assert ratio > 0.2, ratio  # the term is not loose by more than a small factor on single products
    # dot products: the split error sums within TC32_SPLIT * sum |x||w| (the layer bound's zabs term)
    dot_err = (_emulate_3xtf32(x, w).sum(1) - exact.sum(1)).abs()
    assert bool((dot_err <= port_ops.TC32_SPLIT * mag.sum(1)).all())


def test_3xtf32_without_a_correction_product_exceeds_the_split_term():
    x, w = _operands(256, 512, seed=3)
    mag = (x.double() * w.double()).abs().sum(1)
    for drop in ('lh', 'hl'):
        err = (_emulate_3xtf32(x, w, drop=drop).sum(1) - (x.double() * w.double()).sum(1)).abs()
        assert float((err / (port_ops.TC32_SPLIT * mag)).max()) > 20, drop


def test_wide_layer_bound_holds_for_fp32_evaluations():
    """layer_bound('fp32' / 'tf32x3') on EfficientNetV2-tiny ops: the layer evaluated in fp32 (conv2d on the CPU, the
    activation in fp32) lies within the bound; the same values with SiLU's output replaced by its input do not; the
    'tf32x3' bound of a tc32-eligible op is the 'fp32' bound plus exactly TC32_SPLIT * zabs."""
    pcfg = port.PathConfig(proc_side=64)
    spec = port.effnet_spec('efficientnetv2-tiny')
    sd = port.make_effnet_state_dict(spec, pcfg, 8, seed=0, calib_batch=1)
    table = port_ops.effnet_op_table(spec)
    g = torch.Generator().manual_seed(4)
    checked = 0
    for name, op in table.items():
        if op['stem'] or op['depthwise'] or op['act'] != 'silu' or op['kernel'] != 1:
            continue
        cin = sd[op['weight']].shape[1]
        x = torch.randn(2, 8, 8, cin, generator=g).double()
        for precision in ('fp32', 'tf32x3'):
            ref, tol = port_ops.layer_bound(sd, spec, name, x, precision=precision)
            dev = port_ops.conv_layer_reference(sd, spec, name, x.float(), precision=precision, dtype=torch.float32)
            worst, bad = port_ops.check_bound(dev, ref, tol, precision)
            assert bad == 0, (name, precision, worst)
            w, b = (t.float() for t in port_ops._fold(sd, op))
            z = F.conv2d(x.float().permute(0, 3, 1, 2), w, b).permute(0, 2, 3, 1)
            assert port_ops.check_bound(z, ref, tol, precision)[1] > 0, (name, precision)
        assert port_ops.tc32_eligible(op, cin, sd[op['weight']].shape[0])
        _, tol32 = port_ops.layer_bound(sd, spec, name, x, precision='fp32')
        _, tol3x = port_ops.layer_bound(sd, spec, name, x, precision='tf32x3')
        assert bool((tol3x > tol32).all())
        checked += 1
        if checked == 3:
            break
    assert checked == 3


def test_pool_mean_bound_holds_for_the_kernel_order():
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(3, 17, 13, 64, generator=g) * 100).float()
    mean, tol = port_ops.pool_mean_bound(x)
    p = x.shape[1] * x.shape[2]
    flat = x.reshape(3, p, 64)
    part = torch.zeros(8, 3, 64, dtype=torch.float32)
    for px in range(p):  # per-thread strided sums (threadIdx.y = px % 8), then the 8-way tree, then * (1/P) in fp32
        part[px % 8] = part[px % 8] + flat[:, px]
    s = part[0]
    for i in range(1, 8):
        s = s + part[i]
    dev = s * torch.tensor(1.0 / p, dtype=torch.float32)
    assert bool(((dev.double() - mean).abs() <= tol).all())
    wrong = (s - part[7]) * torch.tensor(1.0 / p, dtype=torch.float32)  # one slice left out
    assert bool(((wrong.double() - mean).abs() > tol).any())


def _decode_case(seed, b=3, j=5, depth=8, hw=8):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(b, j * (1 + depth), hw, hw, generator=g, dtype=torch.float64) * 3
    delta = torch.rand(b, j * (1 + depth), hw, hw, generator=g, dtype=torch.float64) * 1e-3
    return logits, delta


def _decode(logits, cfg, j):
    l2, l3 = port.split_logits(logits, j, cfg.depth)
    c2 = port.heatmap_to_image(port.soft_argmax(l2, dims=(3, 2)), cfg)
    c3 = port.heatmap_to_metric(port.soft_argmax(l3, dims=(4, 3, 1)), cfg)
    return c2, c3


def test_decode_bound_holds_for_perturbed_logits():
    cfg = port.PathConfig(proc_side=256, depth=8)
    j = 5
    for seed in range(3):
        logits, delta = _decode_case(seed, j=j, depth=cfg.depth)
        c2, t2, c3, t3 = port_ops.decode_bound(logits, delta, cfg, j)
        r2, r3 = _decode(logits, cfg, j)
        assert torch.allclose(c2, r2, rtol=0, atol=1e-9) and torch.allclose(c3, r3, rtol=0, atol=1e-9)
        # the worst direction per coordinate: logits above the coordinate raised by delta, the others lowered
        for sign in (1.0, -1.0):
            g = torch.Generator().manual_seed(100 + seed)
            rnd = logits + delta * (2 * torch.rand(logits.shape, generator=g, dtype=torch.float64) - 1)
            xs = port.linspace01(logits.shape[-1], torch.float64)
            tilt = logits + sign * delta * torch.sign(xs - 0.5)[None, None, None, :]
            for pert in (rnd, tilt):
                p2, p3 = _decode(pert, cfg, j)
                assert bool(((p2 - c2).abs() <= t2).all()), float(((p2 - c2).abs() / t2).max())
                assert bool(((p3 - c3).abs() <= t3).all()), float(((p3 - c3).abs() / t3).max())
        assert float(t2.max()) < 0.5 and float(t3.max()) < 5.0  # well under a pixel / a few mm at this delta


def test_decode_bound_rejects_a_misweighted_column():
    """the decode with the last column of every fourth pixel weighted x + 1 (an off-by-one in one pixel slice)."""
    cfg = port.PathConfig(proc_side=256, depth=8)
    j = 5
    logits, delta = _decode_case(7, j=j, depth=cfg.depth)
    c2, t2, _c3, _t3 = port_ops.decode_bound(logits, delta, cfg, j)
    l2 = port.split_logits(logits, j, cfg.depth)[0]
    e = torch.exp(l2 - l2.amax(dim=(2, 3), keepdim=True))
    w = l2.shape[-1]
    xi = torch.arange(w, dtype=torch.float64).expand(l2.shape[2], w).clone()
    pix = torch.arange(l2.shape[2] * w).reshape(l2.shape[2], w)
    xi[(pix % 4 == 3) & (xi == w - 1)] += 1
    x = (e * xi).sum(dim=(2, 3)) / e.sum(dim=(2, 3)) / (w - 1)
    px = x * float(255 - 255 % cfg.stride_test) + cfg.stride_test // 2
    assert bool(((px - c2[..., 0]).abs() > t2[..., 0]).any())
