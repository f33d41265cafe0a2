"""`-m gpu` checks of every kernel that reduces a row or a group -- GroupNorm, LayerNorm, the folded LayerNorm and the
softmaxes -- against float64 on ill-conditioned inputs: large common offsets (mean/std up to 1000), offsets that
alternate sign per group, real per-channel offsets, exactly constant groups, std far below sqrt(eps) and far above 1,
sharp softmaxes whose dominant key arrives in the last key block.

Every reference is float64 torch on the same 16-bit-rounded inputs the kernel reads (upcast), with the same fp32
gamma / beta / weights.  u is the unit roundoff of the storage type (2^-11 fp16, 2^-8 bf16).  Each bound is stated
once below as a formula; it covers the 16-bit rounding of the output (and of P in attention) with a factor of two to
spare, while the kernels' fp32 statistics, when right, are ~1e-5 relative.  An excess therefore means a statistic is
wrong.  Every case prints its worst err / bound ratio.
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
U = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}
# half the smallest subnormal: the absolute part of rounding a value near 0 to the storage type
ETA = {"fp16": 2.0 ** -25, "bf16": 2.0 ** -134}
# common offsets r = mean / std: as far as each format still resolves std-1 data (fp16 at 1000: a step is 0.5 std)
OFFSETS = {"fp16": (0, 30, 100, 300, 1000), "bf16": (0, 30, 100)}


@pytest.fixture(params=list(DTYPES))
def storage(request, cuda_device):
    from instancediffusion_b200 import ops
    with ops.storage(DTYPES[request.param]):
        yield request.param


def _ops():
    from instancediffusion_b200 import ops
    return ops


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def _report(what, err, bound):
    """Print the worst err / bound ratio; return a failure message or None."""
    ratio = (err / bound).max().item()
    print(f"[{what}] worst err/bound = {ratio:.3f}")
    if not math.isfinite(ratio) or ratio > 1.0:
        return f"{what}: worst err/bound {ratio:.3g}"
    return None


def _finish(fails):
    assert not fails, "\n".join(fails)


# --------------------------------------------------------------------------------------------
# normalisation inputs: families of (rows, C) tensors whose "units" are GroupNorm groups or LayerNorm rows.  `unit`
# (the group of each channel, or the index of each row) selects the units whose offset alternates in sign or which
# are held constant.
# --------------------------------------------------------------------------------------------
def _families(storage):
    r_max = OFFSETS[storage][-1]
    fams = [(f"offset {r}", "offset", r) for r in OFFSETS[storage]]
    fams += [(f"alternating +-{r_max}", "alternate", r_max),
             (f"per-channel offsets in +-{r_max}", "per_channel", r_max),
             (f"constant units at {r_max + 0.5}", "constant", r_max + 0.5),  # exactly representable in both formats
             ("std 1e-3", "scale", 1e-3),
             ("std 1e3", "scale", 1e3)]
    return fams


def _family_input(kind, r, shape, unit, gen, dt):
    """shape (..., C) float32 on the generator's device; unit: int tensor broadcastable to shape (group / row id)."""
    dev = gen.device
    x = torch.randn(shape, generator=gen, device=dev)
    if kind == "offset":
        x += r
    elif kind == "alternate":
        x += r * (1.0 - 2.0 * (unit % 2)).float()
    elif kind == "per_channel":
        x += r * (2.0 * torch.rand(shape[-1], generator=gen, device=dev) - 1.0)
    elif kind == "constant":
        x += r
        x = torch.where(unit % 4 == 1, torch.full_like(x, r), x)
    elif kind == "scale":
        x *= r
    return x.to(dt)


def _gamma_beta(C, device, seed):
    g = _gen(device, seed)
    gamma = 1.0 + 0.2 * torch.randn(C, generator=g, device=device)
    beta = 0.5 * torch.randn(C, generator=g, device=device)
    return gamma, beta


def _norm_bound(u, t64, gamma):
    # |y - y64| <= 2u (|t64| + |gamma|), t64 = float64 value before SiLU
    return 2.0 * u * (t64.abs() + gamma.double().abs())


# --------------------------------------------------------------------------------------------
# 1a. GroupNorm
# --------------------------------------------------------------------------------------------
GN_UNET = [(2, 4096, 320), (2, 1024, 640), (3, 64, 2560), (8, 256, 1280)]
GN_VAE = [(1, 4096, 512), (1, 65536, 256), (1, 262144, 128)]
GN_GROUPS = 32


def _groupnorm_t64(x, B, HW, C, gamma, beta, eps):
    xd = x.double().view(B, HW, GN_GROUPS, C // GN_GROUPS)
    mean = xd.mean(dim=(1, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    t = (xd - mean) / torch.sqrt(var + eps)
    return t.view(B * HW, C) * gamma.double() + beta.double()


@pytest.mark.parametrize("path", ["single_pass", "two_kernel", "batch_invariant"])
@pytest.mark.parametrize("B,HW,C", GN_UNET + GN_VAE)
def test_groupnorm_conditioning(storage, cuda_device, B, HW, C, path):
    """The default dispatch (single-pass cluster kernel where the launch fits one wave), the forced two-kernel path
    and batch-invariant mode, with and without SiLU, at eps 1e-5 and 1e-6 (VAE decoder shapes: 1e-6)."""
    ops = _ops()
    u = U[storage]
    gamma, beta = _gamma_beta(C, cuda_device, 11)
    unit = (torch.arange(C, device=cuda_device) // (C // GN_GROUPS))[None, :]
    epss = (1e-6,) if (B, HW, C) in GN_VAE else (1e-5, 1e-6)
    fails = []
    if path == "two_kernel":
        os.environ["IDIFF_GN_FUSED"] = "0"
    elif path == "batch_invariant":
        ops.set_batch_invariant(True)
    try:
        for i, (name, kind, r) in enumerate(_families(storage)):
            x = _family_input(kind, r, (B * HW, C), unit, _gen(cuda_device, 100 + i), DTYPES[storage])
            for eps in epss:
                t64 = _groupnorm_t64(x, B, HW, C, gamma, beta, eps)
                bound = _norm_bound(u, t64, gamma)
                for silu in (False, True):
                    y = ops.groupnorm(x, gamma, beta, batch=B, hw=HW, groups=GN_GROUPS, eps=eps, silu=silu)
                    y64 = F.silu(t64) if silu else t64
                    err = (y.double() - y64).abs()
                    fails.append(_report(f"groupnorm {path} {storage} B{B} HW{HW} C{C} eps{eps:g} silu={silu} {name}",
                                         err, bound))
    finally:
        os.environ.pop("IDIFF_GN_FUSED", None)
        ops.set_batch_invariant(False)
    _finish([f for f in fails if f])


# --------------------------------------------------------------------------------------------
# 1b. LayerNorm (two-pass; a constant row must give exactly beta, so the mean is s / C, not s * fl(1 / C))
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [320, 640, 1280, 96, 384, 768])  # fast path, then the generic one-warp-per-row path
def test_layernorm_conditioning(storage, cuda_device, C):
    ops = _ops()
    u = U[storage]
    rows = 1003
    gamma, beta = _gamma_beta(C, cuda_device, 12)
    unit = torch.arange(rows, device=cuda_device)[:, None]
    fails = []
    for i, (name, kind, r) in enumerate(_families(storage)):
        x = _family_input(kind, r, (rows, C), unit, _gen(cuda_device, 200 + i), DTYPES[storage])
        xd = x.double()
        for eps in (1e-5, 1e-6):
            mean = xd.mean(-1, keepdim=True)
            var = ((xd - mean) ** 2).mean(-1, keepdim=True)
            t64 = (xd - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()
            y = ops.layernorm(x, gamma, beta, eps)
            fails.append(_report(f"layernorm {storage} C{C} eps{eps:g} {name}", (y.double() - t64).abs(),
                                 _norm_bound(u, t64, gamma)))
    _finish([f for f in fails if f])


# --------------------------------------------------------------------------------------------
# 1c. folded LayerNorm: row statistics from a producer GEMM's epilogue or from row_stats, consumed by a plain and a
# GEGLU GEMM.  The (sum, sum of squares) slot format is accurate to about r = 30; r = 100 and 300 are measured and
# printed only (their errors are recorded in the fold_layernorm / RowStats docstrings).
# --------------------------------------------------------------------------------------------
FOLD_ASSERTED = (0, 30)
FOLD_MEASURED = (100, 300)


def _gelu64(g):
    return 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0)))


@pytest.mark.parametrize("C", [320, 640, 1280])
def test_layernorm_fold_conditioning(storage, cuda_device, C):
    """Reference: float64 LayerNorm of the stored x, then the linear layer with the folded weights the kernel reads
    (fold_layernorm's 16-bit W * gamma and fp32 W beta + b).  Bound, with M = |xhat64| |w|^T the magnitude of the
    products: plain |y - y64| <= 2u |y64| + u M; GEGLU y = v gelu(g):
    |y - y64| <= 2u |y64| + u (M_v |gelu(g64)| + 1.13 |v64| M_g) (1.13 = max |gelu'|)."""
    from instancediffusion_b200.packing import GEGLU_GROUP, pack_geglu
    ops = _ops()
    u = U[storage]
    dt = DTYPES[storage]
    M, eps = 1000, 1e-5
    g = _gen(cuda_device, 13)
    a = torch.randn((M, C), generator=g, device=cuda_device).to(dt)
    w0 = (torch.randn((C, C), generator=g, device=cuda_device) / math.sqrt(C)).to(dt)
    res = torch.randn((M, C), generator=g, device=cuda_device).to(dt)
    gamma = 1.0 + 0.3 * torch.randn(C, generator=g, device=cuda_device)
    beta = 0.2 * torch.randn(C, generator=g, device=cuda_device)
    w1 = torch.randn((3 * C, C), generator=g, device=cuda_device) / math.sqrt(C)
    wg = torch.randn((8 * C, C), generator=g, device=cuda_device) / math.sqrt(C)
    bg = 0.3 * torch.randn(8 * C, generator=g, device=cuda_device)
    b0n = 0.3 * torch.randn(C, generator=g, device=cuda_device)
    f1 = ops.fold_layernorm(w1, None, gamma, beta, eps)
    fg = ops.fold_layernorm(wg, bg, gamma, beta, eps, pack=pack_geglu)
    fails = []
    for r in FOLD_ASSERTED + FOLD_MEASURED:
        x, st = ops.gemm(a, w0, b0n + r, residual=res, want_stats=True)  # x ~ r + N(0, 1.4)
        xd = x.double()
        mean = xd.mean(-1, keepdim=True)
        xhat = (xd - mean) / torch.sqrt(((xd - mean) ** 2).mean(-1, keepdim=True) + eps)
        # plain consumer
        w1d = f1.w.double()
        y1 = xhat @ w1d.t() + f1.bias.double()
        b1 = 2 * u * y1.abs() + u * (xhat.abs() @ w1d.abs().t())
        # GEGLU consumer (pack_geglu interleaves value / gate rows in groups of GEGLU_GROUP)
        wgd = fg.w.double()
        h = xhat @ wgd.t() + fg.bias.double()
        hm = xhat.abs() @ wgd.abs().t()
        nt = h.shape[1] // (2 * GEGLU_GROUP)
        v, gt = (t.reshape(M, nt, 2, GEGLU_GROUP) for t in (h, hm))
        v64, g64 = v[:, :, 0].reshape(M, -1), v[:, :, 1].reshape(M, -1)
        mv, mg = gt[:, :, 0].reshape(M, -1), gt[:, :, 1].reshape(M, -1)
        yg = v64 * _gelu64(g64)
        bgd = 2 * u * yg.abs() + u * (mv * _gelu64(g64).abs() + 1.13 * v64.abs() * mg)
        for src, s in (("producer stats", st), ("row_stats", ops.row_stats(x))):
            out1 = ops.gemm(x, f1.w, f1.bias, ln=(s, f1.colsum, f1.eps))
            outg = ops.gemm(x, fg.w, fg.bias, geglu=True, ln=(s, fg.colsum, fg.eps))
            for cons, out, ref, bound in (("plain", out1, y1, b1), ("geglu", outg, yg, bgd)):
                err = (out.double() - ref).abs()
                what = f"ln-fold {storage} C{C} r{r} {src} {cons}"
                msg = _report(what, err, bound)
                if r in FOLD_MEASURED:
                    print(f"[{what}] (documented range only) max|err| / max|y64| = "
                          f"{(err.max() / ref.abs().max()).item():.3e}")
                else:
                    fails.append(msg)
    _finish([f for f in fails if f])


# --------------------------------------------------------------------------------------------
# 1d. softmaxes.  Bound, row-wise: |O - O64| <= 4u (P64 |V|) + u |O64| + eta, eta the absolute rounding floor of
# the 16-bit output (an fp16 O below 2^-14 is subnormal; a row dominated by one key whose |v| is tiny gets there);
# softmax_rows_: |p - p64| <= 2u p64 + 2^-24.  References are taken per batch entry so float64 scores stay small.
# --------------------------------------------------------------------------------------------
def _attn_bound(storage, pv64, o64):
    # pv64 = P64 |V|
    return 4.0 * U[storage] * pv64 + U[storage] * o64.abs() + ETA[storage]


N_OBJ, N_CTX, HEADS = 184, 77, 8
# the dominant key in the last block of segment 0 (a ragged block when n0 is not a block multiple), or segment 1
PEAKS = {"self": (None, "seg0"), "cross": (None, "seg0"), "gated": (None, "seg0", "seg1")}
ATTN_CASES = [(kind, peak) for kind, peaks in PEAKS.items() for peak in peaks]
PEAK_MARGIN = 10.0  # natural-log units above the largest other score the row can expect (4 S)


def _attn_inputs(kind, B, nq, d, S, peak, dt, device, seed):
    """q scaled so the scores have std S.  With a peak, coordinate 0 of every head is 8 in the even query rows and 0
    in the odd ones, and only the peak key has a non-zero coordinate 0, sized so that its score in the even rows is
    4 S + PEAK_MARGIN."""
    g = _gen(device, seed)
    C = HEADS * d
    n0 = N_CTX if kind == "cross" else nq
    n1 = N_OBJ if kind == "gated" else 0
    q = torch.randn((B, nq, HEADS, d), generator=g, device=device) * S
    k = torch.randn((B, n0 + n1, HEADS, d), generator=g, device=device)
    v = torch.randn((B, n0 + n1, HEADS, d), generator=g, device=device)
    if peak is not None:
        j = n0 - 1 if peak == "seg0" else n0 + n1 - 1
        k[:, :, :, 0] = 0.0
        q[:, :, :, 0] = 0.0
        q[:, 0::2, :, 0] = 8.0
        k[:, j, :, 0] = (4.0 * S + PEAK_MARGIN) / (8.0 * d ** -0.5)
    return q.reshape(B * nq, C).to(dt), k.to(dt), v.to(dt), n0, n1


def _attn_ref(q, k, v, B, nq, d, mask=None):
    """float64 (O, P @ |V|) per batch entry: q [B*nq, C], k / v [B, n, H, d]."""
    o, pv = [], []
    for b in range(B):
        qb = q[b * nq:(b + 1) * nq].double().view(nq, HEADS, d).transpose(0, 1)
        kb = k[b].double().transpose(0, 1)
        vb = v[b].double().transpose(0, 1)
        s = (qb @ kb.transpose(-1, -2)) * d ** -0.5
        if mask is not None:
            mq, mk = mask
            allowed = (mq[b][:, None] & mk[b][None, :]) != 0
            idx = torch.arange(nq, device=s.device)
            allowed[idx, idx] = True  # a visual token always sees itself
            s = s.masked_fill(~allowed[None], float("-inf"))
        p = torch.softmax(s, -1)
        o.append((p @ vb).transpose(0, 1).reshape(nq, -1))
        pv.append((p @ vb.abs()).transpose(0, 1).reshape(nq, -1))
    return torch.cat(o), torch.cat(pv)


def _attn_run(q, k, v, B, nq, d, n0, n1, mask=None):
    ops = _ops()
    C = HEADS * d
    k2, v2 = k.reshape(B, -1, C), v.reshape(B, -1, C)
    k0, v0 = k2[:, :n0].reshape(B * n0, C), v2[:, :n0].reshape(B * n0, C)
    kw = {}
    if n1:
        kw = dict(k1=k2[:, n0:].reshape(B * n1, C), v1=v2[:, n0:].reshape(B * n1, C), n1=n1, kv1_batch=B)
    if mask is not None:
        kw["mask"] = mask
    return ops.attention(q, k0, v0, batch=B, heads=HEADS, head_dim=d, nq=nq, n0=n0, scale=d ** -0.5, **kw)


@pytest.mark.parametrize("S", [1, 8, 32])
@pytest.mark.parametrize("nq", [768, 1000])  # a multiple of both query tiles (192 at d = 40, 128 otherwise), and not
@pytest.mark.parametrize("kind,peak", ATTN_CASES)
@pytest.mark.parametrize("d", [40, 80, 160])
def test_attention_conditioning(storage, cuda_device, d, kind, peak, nq, S):
    B = 2
    q, k, v, n0, n1 = _attn_inputs(kind, B, nq, d, S, peak, DTYPES[storage], cuda_device, seed=d + nq + S)
    out = _attn_run(q, k, v, B, nq, d, n0, n1)
    o64, pv64 = _attn_ref(q, k, v, B, nq, d)
    bound = _attn_bound(storage, pv64, o64)
    _finish([m for m in [_report(f"attention d{d} {kind} peak={peak} nq{nq} S{S} {storage}",
                                 (out.double() - o64).abs(), bound)] if m])


@pytest.mark.parametrize("S", [1, 8, 32])
@pytest.mark.parametrize("nq", [768, 1000])
@pytest.mark.parametrize("kind", ["self", "gated"])
def test_attention_masked_late_keys(storage, cuda_device, kind, nq, S):
    """d = 40 with the instance-isolation mask.  Every third query row shares a mask bit only with the last 40 keys of
    segment 0 (and, gated, the last 20 object tokens): its running max sits on its own key until the last blocks."""
    d, B = 40, 2
    q, k, v, n0, n1 = _attn_inputs(kind, B, nq, d, S, None, DTYPES[storage], cuda_device, seed=7 + nq + S)
    g = torch.Generator().manual_seed(nq + S)
    mq = (torch.randint(0, 32, (B, nq), generator=g) & torch.randint(0, 32, (B, nq), generator=g)) << 1
    mq[:, 0::3] = 1
    mk = torch.randint(0, 32, (B, n0 + n1), generator=g) << 1
    mk[:, n0 - 40:n0] |= 1
    if n1:
        mk[:, n0 + n1 - 20:] |= 1
    mask = (mq.to(torch.int32).to(cuda_device).contiguous(), mk.to(torch.int32).to(cuda_device).contiguous())
    out = _attn_run(q, k, v, B, nq, d, n0, n1, mask=mask)
    o64, pv64 = _attn_ref(q, k, v, B, nq, d, mask=mask)
    bound = _attn_bound(storage, pv64, o64)
    _finish([m for m in [_report(f"masked attention d40 {kind} nq{nq} S{S} {storage}",
                                 (out.double() - o64).abs(), bound)] if m])


@pytest.mark.parametrize("S", [1, 8, 32])
@pytest.mark.parametrize("n", [1000, 4096, 4104, 6152])  # 4096 is a multiple of 2048, the others are not
def test_softmax_rows_conditioning(storage, cuda_device, n, S):
    """Logits with std S; every even row has its peak (row max + 10) in the last 16-byte vector."""
    ops = _ops()
    rows = 64
    g = _gen(cuda_device, n + S)
    x = torch.randn((rows, n), generator=g, device=cuda_device) * S
    r = torch.arange(0, rows, 2, device=cuda_device)
    x[r, n - 1 - (r // 2) % 8] = x[r].max(-1).values + 10.0
    x = x.to(DTYPES[storage])
    p64 = torch.softmax(x.double(), -1)
    p = ops.softmax_rows_(x.clone())
    bound = 2.0 * U[storage] * p64 + 2.0 ** -24
    _finish([m for m in [_report(f"softmax_rows n{n} S{S} {storage}", (p.double() - p64).abs(), bound)] if m])


@pytest.mark.parametrize("S", [1, 8, 32])
def test_causal_attention_small_diagonal_peak(storage, cuda_device, S):
    """CLIP text shape (77 tokens, 12 heads of 64): k = k_rand + (S / 8) q, so the score on the diagonal -- the last
    key a causal row sees -- is about S while the others have std about sqrt(1 + (S / 8)^2)."""
    ops = _ops()
    B, T, H, D = 2, 77, 12, 64
    dt = DTYPES[storage]
    g = _gen(cuda_device, 300 + S)
    q = torch.randn((B, T, H, D), generator=g, device=cuda_device)
    k = torch.randn((B, T, H, D), generator=g, device=cuda_device) + (S / 8.0) * q
    v = torch.randn((B, T, H, D), generator=g, device=cuda_device)
    qkv = torch.cat([t.reshape(B * T, H * D) for t in (q, k, v)], 1).to(dt).contiguous()
    out = ops.causal_attention_small(qkv, batch=B, tokens=T, heads=H, head_dim=D, scale=D ** -0.5)
    q64, k64, v64 = (qkv[:, i * H * D:(i + 1) * H * D].double().view(B, T, H, D).transpose(1, 2) for i in range(3))
    s = (q64 @ k64.transpose(-1, -2)) * D ** -0.5
    s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=cuda_device).triu(1), float("-inf"))
    p = torch.softmax(s, -1)
    o64 = (p @ v64).transpose(1, 2).reshape(B * T, H * D)
    pv64 = (p @ v64.abs()).transpose(1, 2).reshape(B * T, H * D)
    bound = _attn_bound(storage, pv64, o64)
    _finish([m for m in [_report(f"causal_attention_small S{S} {storage}", (out.double() - o64).abs(), bound)] if m])
