"""CPU checks of the float64 references in tests/cases_census.py against torch's own functional ops on small tensors,
and of the launch signature: the references judge the kernels in tests/test_launch_census_gpu.py, so they are
tested first."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cases_census as CC  # noqa: E402

TOL = dict(rtol=1e-10, atol=1e-12)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b):
    torch.testing.assert_close(a.double(), b.double(), **TOL)


def test_gemm_reference_epilogues():
    from instancediffusion_b200.packing import pack_geglu
    g = _g(1)
    M, N, K, R = 12, 256, 40, 4
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g)
    b, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    radd, gr = torch.randn(3, N, generator=g), torch.tensor([0.5, 0.0, 2.0])
    lin = F.linear(a.double(), w.double(), b.double())
    y, bound = CC.gemm64(a, w, b)
    _close(y, lin)
    assert (bound >= 2 * CC.U[torch.float16] * lin.abs()).all()
    _close(CC.gemm64(a, w, b, silu=True, rowadd=radd, rows_per_batch=R)[0],
           F.silu(lin + radd.double().repeat_interleave(R, 0)))
    _close(CC.gemm64(a, w, b, gelu=True)[0], F.gelu(lin))
    y, _ = CC.gemm64(a, w, b, residual=res, gate=0.7, gate_rows=gr, rows_per_batch=R)
    _close(y, res.double() + 0.7 * gr.double().repeat_interleave(R)[:, None] * lin)
    assert torch.equal(y[R:2 * R], res[R:2 * R].double())  # a zero gate passes the residual through
    wp, bp = pack_geglu(w, b)
    v, gate = lin.chunk(2, -1)
    _close(CC.gemm64(a, wp, bp, geglu=True)[0], v * F.gelu(gate))


def test_ln_fold_reference_is_layernorm_then_linear():
    """The folded consumer's reference takes no statistics: float64 LayerNorm of the rows, then the folded weights."""
    g = _g(2)
    M, K, N, eps = 9, 64, 24, 1e-5
    x = torch.randn(M, K, generator=g) * 3 + 5
    w, bias = torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    y, bound = CC.gemm64(x, w, bias, ln=(w.sum(1), eps))
    _close(y, F.linear(F.layer_norm(x.double(), (K,), eps=eps), w.double(), bias.double()))
    assert torch.isfinite(bound).all()


def test_conv3x3_reference():
    from instancediffusion_b200.packing import pack_conv3x3
    g = _g(3)
    B, H, W, Cin, Cout = 2, 5, 6, 8, 16
    x = torch.randn(B, Cin, H, W, generator=g)
    wt, b = torch.randn(Cout, Cin, 3, 3, generator=g), torch.randn(Cout, generator=g)
    radd = torch.randn(B, Cout, generator=g)
    nhwc = x.permute(0, 2, 3, 1).reshape(B * H * W, Cin)
    y, _ = CC.gemm64(nhwc, pack_conv3x3(wt), b, conv=(B, H, W, Cin), rowadd=radd)
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1) + radd.double()[:, :, None, None]
    _close(y, ref.permute(0, 2, 3, 1).reshape(B * H * W, Cout))
    _close(CC.unpack_conv3x3(pack_conv3x3(wt)), wt)


def test_slot_check_finds_the_tile_width():
    g = _g(4)
    M, N = 5, 640
    y = torch.randn(M, N, generator=g).half()
    for bn in (128, 160):
        yd = y.double()
        st = torch.stack([torch.stack([yd[:, s:s + bn].sum(1), (yd[:, s:s + bn] ** 2).sum(1)], -1)
                          for s in range(0, N, bn)]).float()
        fits = CC.slot_check(y, st, True, torch.float16)
        assert fits[bn] <= 1.0 and all(r > 1.0 for k, r in fits.items() if k != bn), (bn, fits)
        st[-1, :, 0] -= yd[:, N - 8:].sum(1).float()  # a last 8-column group left out of the sums
        assert CC.slot_check(y, st, True, torch.float16)[bn] > 1.0
    assert CC.slot_check(y, torch.zeros(2, M, 2), True, torch.float16) == {}  # 2 slots: no tile width fits 640


def test_normalisation_and_softmax_references():
    g = _g(5)
    B, HW, C = 2, 10, 64
    x = torch.randn(B * HW, C, generator=g) + 2
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    y, _ = CC.groupnorm64(x, gamma, beta, batch=B, hw=HW, eps=1e-5, silu=True)
    ref = F.silu(F.group_norm(x.double().view(B, HW, C).permute(0, 2, 1), 32, gamma.double(), beta.double(), 1e-5))
    _close(y, ref.permute(0, 2, 1).reshape(B * HW, C))
    _close(CC.layernorm64(x, gamma, beta, 1e-6)[0], F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-6))
    _close(CC.softmax_rows64(x)[0], F.softmax(x.double(), -1))


@pytest.mark.parametrize("mask", [False, True])
def test_attention_reference(mask):
    g = _g(6)
    B, H, d, nq, n1 = 2, 2, 8, 6, 3
    C = H * d
    q, k0, v0 = (torch.randn(B * nq, C, generator=g) for _ in range(3))
    k1, v1 = (torch.randn(n1, C, generator=g) for _ in range(2))
    m = None
    allowed = torch.ones(B, nq, nq + n1, dtype=torch.bool)
    if mask:
        mq = torch.randint(0, 4, (B, nq), generator=g, dtype=torch.int32)
        mk = torch.randint(0, 4, (B, nq + n1), generator=g, dtype=torch.int32)
        m = (mq, mk)
        allowed = (mq[:, :, None] & mk[:, None, :]) != 0
        allowed[:, torch.arange(nq), torch.arange(nq)] = True
    o, _ = CC.attention64(q, k0, v0, batch=B, heads=H, head_dim=d, nq=nq, n0=nq, scale=d ** -0.5, k1=k1, v1=v1,
                          n1=n1, kv1_batch=1, mask=m)
    heads = lambda t, n: t.double().view(-1, n, H, d).transpose(1, 2)  # noqa: E731
    kk = torch.cat([heads(k0, nq), heads(k1, n1).expand(B, H, n1, d)], 2)
    vv = torch.cat([heads(v0, nq), heads(v1, n1).expand(B, H, n1, d)], 2)
    ref = F.scaled_dot_product_attention(heads(q, nq), kk, vv, attn_mask=allowed[:, None])
    _close(o, ref.transpose(1, 2).reshape(B * nq, C))


def test_scaleu_reference_is_the_fft_filter():
    """ScaleU's skip half against torch.fft in complex128 directly: x + (s - 1) * the centre 2x2 of the shifted
    spectrum."""
    g = _g(7)
    B, H, W, c1, c2, s = 2, 6, 8, 8, 16, 1.3
    h, skip = torch.randn(B * H * W, c1, generator=g), torch.randn(B * H * W, c2, generator=g) + 0.5
    b1 = torch.rand(c1, generator=g) + 0.5
    y, _ = CC.scaleu64(h, skip, b1, s, batch=B, height=H, width=W)
    _close(y[:, :c1], h.double() * b1.double())
    xs = skip.double().view(B, H, W, c2).permute(0, 3, 1, 2)
    f = torch.fft.fftshift(torch.fft.fft2(xs), dim=(-2, -1))
    low = torch.zeros_like(f)
    low[..., H // 2 - 1:H // 2 + 1, W // 2 - 1:W // 2 + 1] = f[..., H // 2 - 1:H // 2 + 1, W // 2 - 1:W // 2 + 1]
    ref = xs + (s - 1) * torch.fft.ifft2(torch.fft.ifftshift(low, dim=(-2, -1))).real
    _close(y[:, c1:], ref.permute(0, 2, 3, 1).reshape(B * H * W, c2))


def test_small_kernel_references():
    from instancediffusion_b200.packing import pack_conv3x3_taps
    g = _g(8)
    B, H, W, C = 2, 6, 4, 8
    x = torch.randn(B, H, W, C, generator=g).half().reshape(B * H * W, C)
    xn = x.double().view(B, H, W, C).permute(0, 3, 1, 2)
    w49, bias = torch.randn(49, C, generator=g), torch.randn(C, generator=g)
    ref = F.conv2d(xn, w49.double().t().reshape(C, 1, 7, 7), bias.double(), padding=3, groups=C)
    _close(CC.dwconv7x7_64(x, w49, bias, B, H, W)[0], ref.permute(0, 2, 3, 1).reshape(-1, C))
    cols = CC.im2col_s2_ref(x, B, H, W)
    wt = torch.randn(5, C, 3, 3, generator=g)
    from instancediffusion_b200.packing import pack_conv3x3
    ref = F.conv2d(xn, wt.double(), stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, 5)
    _close(cols.double() @ pack_conv3x3(wt).double().t(), ref)
    ref = F.conv2d(F.pad(xn, (0, 1, 0, 1)), wt.double(), stride=2).permute(0, 2, 3, 1).reshape(-1, 5)
    _close(CC.im2col_s2_ref(x, B, H, W, pad01=True).double() @ pack_conv3x3(wt).double().t(), ref)
    up = F.interpolate(xn, scale_factor=2, mode="nearest").permute(0, 2, 3, 1).reshape(-1, C)
    _close(CC.upsample_nearest2x_ref(x, B, H, W), up)
    z = torch.randn(B, 4, H, W, generator=g)
    w0, w1 = torch.randn(16, 4, 3, 3, generator=g), torch.randn(16, 4, 3, 3, generator=g)
    b0, b1 = torch.randn(16, generator=g), torch.randn(16, generator=g)
    y, _ = CC.conv_in_select64(z, pack_conv3x3_taps(w0), b0, pack_conv3x3_taps(w1), b1, torch.tensor([0, 1]))
    zr = z.half().double()
    ref = torch.cat([F.conv2d(zr[:1], w0.double(), b0.double(), padding=1),
                     F.conv2d(zr[1:], w1.double(), b1.double(), padding=1)])
    _close(y, ref.permute(0, 2, 3, 1).reshape(-1, 16))
    t = torch.tensor([981.0, 1.0])
    emb, _ = CC.timestep_embedding64(t, 16)
    f = torch.exp(-math.log(10000) * torch.arange(8, dtype=torch.float64) / 8)
    _close(emb, torch.cat([torch.cos(t.double()[:, None] * f), torch.sin(t.double()[:, None] * f)], -1))


def test_signature_tells_kernels_apart():
    from instancediffusion_b200 import ops
    a, w = torch.zeros(256, 64, dtype=torch.float16), torch.zeros(128, 64, dtype=torch.float16)
    res = torch.zeros(256, 128, dtype=torch.float16)
    st = ops.RowStats(torch.zeros(1, 256, 2), 1)

    def sig(invariant=False, storage=torch.float16, **kw):
        base = dict(a=a, w=w, bias=None, residual=None, gate=1.0, gate_rows=None, want_stats=False, ln=None,
                    geglu=False, silu=False, conv=None)
        base.update(kw)
        return CC.signature("gemm", (), base, invariant=invariant, storage=storage)

    variants = [sig(), sig(invariant=True), sig(storage=torch.bfloat16), sig(want_stats=True), sig(geglu=True),
                sig(silu=True), sig(residual=res), sig(residual=res, gate=0.0), sig(residual=res, gate=0.5),
                sig(residual=res, gate_rows=torch.ones(2)), sig(residual=res, gate_rows=torch.tensor([1.0, 0.0])),
                sig(ln=(st, torch.zeros(128), 1e-5)), sig(conv=(1, 16, 16, 64)), sig(a=a[:, :32]),
                sig(a=torch.zeros(512, 64, 2, dtype=torch.float16)[:, :, 0]),
                sig(bias=torch.zeros(128))]
    assert len(set(variants)) == len(variants)
    # values of tensors and of float scalars other than the gate do not split a signature
    assert sig(a=torch.ones(256, 64, dtype=torch.float16), residual=res, gate=0.3) == sig(residual=res, gate=0.7)
    assert (CC.signature("layernorm", (), dict(x=a, eps=1e-5), invariant=False, storage=torch.float16) ==
            CC.signature("layernorm", (), dict(x=a, eps=1e-6), invariant=False, storage=torch.float16))
