"""Float64 restatements of the kernel entry points the model launches, and the error bound of each, for the launch
census (tests/test_launch_census_gpu.py; the references are checked against torch's own ops on the CPU by
tests/test_launch_census_cpu.py).

Every reference takes the recorded inputs of one launch -- the 16-bit tensors the kernel read, upcast -- and returns
the float64 result y64 and the bound of |y - y64| (or an exact expected value).  u is the unit roundoff of the output
(2^-11 fp16, 2^-8 bf16, 2^-24 fp32), e = 2^-24 the fp32 one, eta half the smallest 16-bit subnormal.  The bounds,
each stated once:

  GEMM / conv3x3 (K = depth, 9 Cin for the conv):   |y - y64| <= 2u |y64| + 2 K e Mag + eta
      z = A W^T + bias (+ rowadd), y = residual + gate * gate_row * act(z); GEGLU y = v gelu(g)
      Mag = |gate gate_row| act' (|A| |W|^T + |bias| + |rowadd|) + |residual|, act' = 1, 1.1 (SiLU), 1.13 (GELU)
      GEGLU: Mag = Mag_v |gelu(g64)| + 1.13 |v64| Mag_g
  LayerNorm-folded consumer (reference: float64 LayerNorm of the A rows, then the folded linear layer):
      the GEMM bound with Mag = rstd |x| |w|^T, plus u (1 + E[x^2] / var) |y64 - bias| + u rstd mean|x| |colsum|:
      the producer statistics of the default mode are sums of the values before their 16-bit rounding
  producer statistics, per slot s (columns [s BN, (s + 1) BN) of the stored output y):
      |sum_s - sum y| <= (r + 2 BN e) sum |y|,  |sumsq_s - sum y^2| <= (2r + 2 BN e) sum y^2,
      r = 0 in batch-invariant mode (sums of the stored values), u in the default mode
  attention:  |O - O64| <= 4u (P64 |V|) + u |O64| + eta            (tests/test_conditioning_gpu.py)
  GroupNorm / LayerNorm:  |y - y64| <= 2u (|t64| + |gamma|), t64 the value before SiLU   (ditto)
  softmax_rows_:  |p - p64| <= 2u p64 + e                           (ditto)
  ScaleU:  |y - y64| <= 2u |y64| + 2 e (|x| + 8 |s - 1| sum_plane |x|) + eta  (seven fp32 plane sums, fp32 twiddles)
  sin / cos embeddings:  |y - y64| <= 2u |y64| + e (8 |arg| + 4) + eta
  depthwise 7x7, the input convs, the VAE latent prologue: the GEMM bound with their K
  layout / gather ops (im2col, upsample, patchify, NCHW -> NHWC): exact
"""
import math
import torch
import torch.nn.functional as F

E32 = 2.0 ** -24
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: E32}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 2.0 ** -150}
GEGLU_GROUP = 128  # packing.GEGLU_GROUP: value / gate rows interleaved per 128
GN_GROUPS = 32
BNS = (256, 192, 160, 128)  # the GEMM tile widths


def gelu64(g):
    return 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0)))


# --------------------------------------------------------------------------------------------
# launch signatures
# --------------------------------------------------------------------------------------------
def _norm(v):
    """The part of an argument that selects a kernel or a configuration: shapes, strides, types, flags and integer
    sizes; not the values of tensors or of float scalars."""
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype).replace("torch.", ""))
    if hasattr(v, "slots") and hasattr(v, "t"):  # ops.RowStats
        return ("RowStats", int(v.slots), tuple(v.t.shape))
    if isinstance(v, (list, tuple)):
        return tuple(_norm(x) for x in v)
    if isinstance(v, bool) or v is None or isinstance(v, str):
        return v
    if isinstance(v, int):
        return int(v)
    if isinstance(v, float):
        return "f"
    return type(v).__name__


def signature(op: str, args: tuple, kwargs: dict, *, invariant: bool, storage: torch.dtype):
    """Hashable signature of one launch: op, every argument's shape / stride / type / flag, the mode and the storage
    type.  A GEMM adds what selects its epilogue from values: the gate (0, 1 or other), and whether gate_rows holds a
    zero."""
    extra = ()
    if op == "gemm":
        g = float(kwargs.get("gate", 1.0))
        extra = (("gate", "0" if g == 0 else "1" if g == 1 else "g"),)
        gr = kwargs.get("gate_rows")
        if gr is not None:
            extra += (("gate_rows_zero", bool((gr == 0).any())),)
    return (op, str(storage).replace("torch.", ""), bool(invariant), _norm(tuple(args)),
            tuple(sorted((k, _norm(v)) for k, v in kwargs.items())), extra)


# --------------------------------------------------------------------------------------------
# GEMM / conv3x3
# --------------------------------------------------------------------------------------------
def unpack_conv3x3(w):
    """packing.pack_conv3x3 undone: (Cout, 9 Cin), k = (ky 3 + kx) Cin + c -> (Cout, Cin, 3, 3)."""
    n, k9 = w.shape
    return w.reshape(n, 3, 3, k9 // 9).permute(0, 3, 1, 2)


def unpack_geglu_rows(h):
    """[..., N] in pack_geglu's interleaved column order -> (value [..., N/2], gate [..., N/2]) in chunk(2) order."""
    lead, n = h.shape[:-1], h.shape[-1]
    t = h.reshape(*lead, n // (2 * GEGLU_GROUP), 2, GEGLU_GROUP)
    return t[..., 0, :].reshape(*lead, n // 2), t[..., 1, :].reshape(*lead, n // 2)


def _matmul(a, w, conv):
    """a @ w^T, or the 3x3 padding-1 convolution of NHWC a (conv = (B, H, W, Cin)) with packed w; rows in a's order."""
    if conv is None:
        return a @ w.t()
    B, H, W, Cin = conv
    x = a.reshape(B, H, W, Cin).permute(0, 3, 1, 2)
    y = F.conv2d(x, unpack_conv3x3(w), padding=1)
    return y.permute(0, 2, 3, 1).reshape(B * H * W, -1)


def _entries(M, conv, rows_per_batch):
    """Batch entry of every output row (an image for the conv; else row // rows_per_batch)."""
    per = conv[1] * conv[2] if conv is not None else (rows_per_batch if rows_per_batch > 0 else M)
    return torch.arange(M) // per


def ln_fold_rows(x, eps):
    """float64 LayerNorm without affine of the rows of x: (xhat, mean, rstd, E[x^2] / var)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    return (xd - mean) * rstd, mean, rstd, (xd * xd).mean(-1, keepdim=True) / (var + eps)


def gemm64(a, w, bias=None, *, residual=None, gate=1.0, rowadd=None, rows_per_batch=0, geglu=False, silu=False,
           gelu=False, conv=None, gate_rows=None, ln=None, out_dtype=torch.float16):
    """(y64, bound) of ops.gemm on the recorded inputs; rows in a's row order, columns the output's (N / 2 for GEGLU).
    ln = (colsum, eps): a is the LayerNorm-folded consumer's un-normalised stream.  The fp32 NCHW output is returned
    in NHWC row order like the others."""
    u = U[out_dtype]
    a, w = a.double(), w.double()
    a2 = a.reshape(-1, a.shape[-1]) if conv is None else a.reshape(-1, conv[3])
    M, N = a2.shape[0], w.shape[0]
    K = w.shape[1]
    ent = _entries(M, conv, rows_per_batch)
    b = torch.zeros(N, dtype=torch.float64) if bias is None else bias.double().cpu()
    b = b.to(a.device)
    fold = None
    if ln is not None:
        colsum, eps = ln
        xhat, mean, rstd, m2v = ln_fold_rows(a2, eps)
        z = xhat @ w.t() + b
        mag = rstd * (a2.abs() @ w.abs().t()) + b.abs()
        fold = u * m2v * (z - b).abs() + u * rstd * a2.abs().mean(-1, keepdim=True) * colsum.double().abs()
    else:
        z = _matmul(a2, w, conv) + b
        mag = _matmul(a2.abs(), w.abs(), conv) + b.abs()
    if geglu:
        v, g = unpack_geglu_rows(z)
        mv, mg = unpack_geglu_rows(mag)
        y = v * gelu64(g)
        mag = mv * gelu64(g).abs() + 1.13 * v.abs() * mg
        if fold is not None:
            fv, fg = unpack_geglu_rows(fold)
            fold = fv * gelu64(g).abs() + 1.13 * v.abs() * fg
    else:
        if rowadd is not None:
            ra = rowadd.double()[ent.to(rowadd.device)]
            z = z + ra
            mag = mag + ra.abs()
        if silu:
            y, mag = F.silu(z), 1.1 * mag
        elif gelu:
            y, mag = gelu64(z), 1.13 * mag
        else:
            y = z
    if residual is not None:
        g = torch.full((M, 1), float(gate), dtype=torch.float64, device=a.device)
        if gate_rows is not None:
            g = g * gate_rows.double()[ent.to(gate_rows.device)][:, None]
        r = residual.double().reshape(M, -1)
        y = r + g * y
        mag = g.abs() * mag + r.abs()
        if fold is not None:
            fold = g.abs() * fold
    bound = 2 * u * y.abs() + 2 * K * E32 * mag + ETA[out_dtype]
    if fold is not None:
        bound = bound + fold
    return y, bound


def slot_check(y, stats, invariant, storage):
    """Producer statistics against the stored output y [M, N]: for every tile width whose column partition has as
    many slots as stats, the worst err / bound over the (sum, sumsq) of every slot.  Returns {BN: ratio}; the BN that
    ran is the one whose partition fits (ratio <= 1)."""
    yd = y.double()
    N = yd.shape[1]
    slots = stats.shape[0]
    r = 0.0 if invariant else U[storage]
    out = {}
    for bn in BNS:
        if (N + bn - 1) // bn != slots:
            continue
        worst = 0.0
        for s in range(slots):
            ys = yd[:, s * bn:(s + 1) * bn]
            got = stats[s].double()
            for q, (ref, mag, rr) in enumerate(((ys.sum(1), ys.abs().sum(1), r), ((ys * ys).sum(1), (ys * ys).sum(1), 2 * r))):
                bound = (rr + 2 * bn * E32) * mag + 1e-30
                err = (got[:, q] - ref).abs()
                worst = max(worst, (err / bound).max().item() if torch.isfinite(got[:, q]).all() else math.inf)
        out[bn] = worst
    return out


# --------------------------------------------------------------------------------------------
# attention, normalisation, softmax, ScaleU
# --------------------------------------------------------------------------------------------
def attention64(q, k0, v0, *, batch, heads, head_dim, nq, n0, scale, k1=None, v1=None, n1=0, kv1_batch=0,
                mask=None, out_dtype=torch.float16):
    """(O64, bound) of ops.attention: q [batch nq, >= C], k0 / v0 [batch n0, >= C], k1 / v1 [kv1_batch n1, >= C];
    the instance-isolation mask lets query i see key j when mask_q[i] & mask_k[j] != 0, and always its own key."""
    C = heads * head_dim
    kb1 = kv1_batch or batch
    outs, bounds = [], []
    for b in range(batch):
        qb = q[b * nq:(b + 1) * nq, :C].double().view(nq, heads, head_dim).transpose(0, 1)
        kk = [k0[b * n0:(b + 1) * n0, :C]]
        vv = [v0[b * n0:(b + 1) * n0, :C]]
        if n1:
            bb = b if kb1 == batch else 0
            kk.append(k1[bb * n1:(bb + 1) * n1, :C])
            vv.append(v1[bb * n1:(bb + 1) * n1, :C])
        kb = torch.cat(kk).double().view(-1, heads, head_dim).transpose(0, 1)
        vb = torch.cat(vv).double().view(-1, heads, head_dim).transpose(0, 1)
        allowed = None
        if mask is not None:
            mq, mk = mask
            allowed = (mq[b].long()[:, None] & mk[b].long()[None, :]) != 0
            idx = torch.arange(nq, device=allowed.device)
            allowed[idx, idx] = True
        o = torch.empty((heads, nq, head_dim), dtype=torch.float64, device=q.device)
        pv = torch.empty_like(o)
        for h in range(heads):  # one head at a time: float64 scores of a 96x96 latent are 680 MB per head
            s = (qb[h] @ kb[h].t()) * scale
            if allowed is not None:
                s = s.masked_fill(~allowed, float("-inf"))
            p = torch.softmax(s, -1)
            o[h] = p @ vb[h]
            pv[h] = p @ vb[h].abs()
        o = o.transpose(0, 1).reshape(nq, C)
        pv = pv.transpose(0, 1).reshape(nq, C)
        outs.append(o)
        bounds.append(4 * U[out_dtype] * pv + U[out_dtype] * o.abs() + ETA[out_dtype])
    return torch.cat(outs), torch.cat(bounds)


def _norm_bound(u, t64, gamma):
    return 2.0 * u * (t64.abs() + gamma.double().abs())


def groupnorm64(x, gamma, beta, *, batch, hw, groups=GN_GROUPS, eps=1e-5, silu=False, out_dtype=torch.float16):
    C = x.shape[-1]
    xd = x.double().reshape(batch, hw, groups, C // groups)
    mean = xd.mean(dim=(1, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    t = ((xd - mean) / torch.sqrt(var + eps)).reshape(batch * hw, C) * gamma.double() + beta.double()
    return (F.silu(t) if silu else t), _norm_bound(U[out_dtype], t, gamma)


def layernorm64(x, gamma, beta, eps=1e-5, out_dtype=torch.float16):
    xd = x.double().reshape(-1, x.shape[-1])
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    t = (xd - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()
    return t, _norm_bound(U[out_dtype], t, gamma)


def softmax_rows64(x, out_dtype=torch.float16):
    p = torch.softmax(x.double(), -1)
    return p, 2 * U[out_dtype] * p + E32


def fourier_filter64(x, scale, threshold=1):
    """openaimodel.py Fourier_filter in complex128 on NCHW x (tests/test_kernels_gpu.py _fourier_filter_ref)."""
    import torch.fft as fft
    B, C, H, W = x.shape
    xf = fft.fftshift(fft.fftn(x.double(), dim=(-2, -1)), dim=(-2, -1))
    mask = torch.ones((B, C, H, W), dtype=torch.float64, device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    xf = fft.ifftshift(xf * mask, dim=(-2, -1))
    return fft.ifftn(xf, dim=(-2, -1)).real


def scaleu64(h, skip, b1, s, *, batch, height, width, out_dtype=torch.float16):
    """[h * b1 | Fourier_filter(skip, s)] in NHWC rows, and the ScaleU bound."""
    u = U[out_dtype]
    hw = height * width
    c2 = skip.shape[-1]
    yh = h.double() * b1.double()
    xs = skip.double().reshape(batch, height, width, c2).permute(0, 3, 1, 2)
    ys = fourier_filter64(xs, float(s)).permute(0, 2, 3, 1).reshape(batch * hw, c2)
    plane = skip.double().abs().reshape(batch, hw, c2).sum(1, keepdim=True).expand(batch, hw, c2).reshape(batch * hw, c2)
    bs = 2 * u * ys.abs() + 2 * E32 * (skip.double().abs() + 8 * abs(float(s) - 1) * plane) + ETA[out_dtype]
    bh = 2 * u * yh.abs() + 2 * E32 * yh.abs() + ETA[out_dtype]
    return torch.cat([yh, ys], 1), torch.cat([bh, bs], 1)


# --------------------------------------------------------------------------------------------
# the small kernels of the model's prologues and of the mask encoder
# --------------------------------------------------------------------------------------------
def _trig_bound(u, y, arg, dt):
    return 2 * u * y.abs() + E32 * (8 * arg.abs() + 4) + ETA[dt]


def timestep_embedding64(t, dim, out_dtype=torch.float16):
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    arg = t.double()[:, None] * freqs[None]
    y = torch.cat([torch.cos(arg), torch.sin(arg)], -1)
    return y, _trig_bound(U[out_dtype], y, torch.cat([arg, arg], -1), out_dtype)


def fourier_embed64(coords, masks, null_pos, *, text=None, null_text=None, mask_mode=0, dropped=False,
                    out_dtype=torch.float16):
    """ops.fourier_embed rows [text | 16 frequencies x (sin, cos) of the D coordinates] and their bound."""
    u = U[out_dtype]
    c = coords.double()
    D = c.shape[1]
    m = masks.double()[:, None]
    freqs = 100.0 ** (torch.arange(16, dtype=torch.float64, device=c.device) / 16)
    args = torch.cat([fr * c for fr in freqs for _ in range(2)], -1)
    emb = torch.cat([f(fr * c) for fr in freqs for f in (torch.sin, torch.cos)], -1)
    if dropped:
        mp = torch.zeros_like(m)
    elif mask_mode == 0:
        mp = m
    else:
        mp = ((c.sum(-1, keepdim=True) + m) > 0).double()
    ye = emb * mp + (1 - mp) * null_pos.double()
    be = _trig_bound(u, ye, args * mp, out_dtype)
    if text is None:
        return ye, be
    yt = text.double() * m + (1 - m) * null_text.double()
    return torch.cat([yt, ye], -1), torch.cat([2 * u * yt.abs() + ETA[out_dtype], be], -1)


def conv_in_select64(x, w0, b0, w1, b1, flags, out_dtype=torch.float16):
    """The per-image input conv on x rounded to the storage type (as the kernel reads it); NHWC rows."""
    B, Cc, H, W = x.shape
    xr = x.to(out_dtype).double()
    ys, ms = [], []
    for b in range(B):
        w, bias = (w0, b0) if int(flags[b]) == 0 else (w1, b1)
        wt = w.double().reshape(3, 3, Cc, -1).permute(3, 2, 0, 1)  # pack_conv3x3_taps undone
        ys.append(F.conv2d(xr[b:b + 1], wt, bias.double(), padding=1))
        ms.append(F.conv2d(xr[b:b + 1].abs(), wt.abs(), bias.double().abs(), padding=1))
    y = torch.cat(ys).permute(0, 2, 3, 1).reshape(B * H * W, -1)
    mag = torch.cat(ms).permute(0, 2, 3, 1).reshape(B * H * W, -1)
    return y, 2 * U[out_dtype] * y.abs() + 2 * 36 * E32 * mag + ETA[out_dtype]


def vae_latent_in64(z, w, bias, inv_scale, out_dtype=torch.float16):
    B, Cc, H, W = z.shape
    zz = z.double().permute(0, 2, 3, 1).reshape(B * H * W, Cc) * inv_scale
    y = torch.zeros((B * H * W, 64), dtype=torch.float64, device=z.device)
    mag = torch.zeros_like(y)
    y[:, :w.shape[0]] = zz @ w.double().t() + bias.double()
    mag[:, :w.shape[0]] = zz.abs() @ w.double().abs().t() + bias.double().abs()
    return y, 2 * U[out_dtype] * y.abs() + 2 * Cc * E32 * mag + ETA[out_dtype]


def dwconv7x7_64(x, w49, bias, batch, h, w, out_dtype=torch.float16):
    C = x.shape[-1]
    xd = x.double().reshape(batch, h, w, C).permute(0, 3, 1, 2)
    wt = w49.double().t().reshape(C, 1, 7, 7)
    y = F.conv2d(xd, wt, bias.double(), padding=3, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    mag = F.conv2d(xd.abs(), wt.abs(), bias.double().abs(), padding=3, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    return y, 2 * U[out_dtype] * y.abs() + 2 * 49 * E32 * mag + ETA[out_dtype]


def segs_inconv64(segs, w, bias, out_size, out_dtype=torch.float16):
    """(y64, bound, seg_sum64, seg_sum bound): Conv2d(Cin, 3, 3, 1, 1) of the nearest resize, NHWC rows."""
    rs = F.interpolate(segs.double(), out_size, mode="nearest")
    Cin = segs.shape[1]
    y = F.conv2d(rs, w.double(), bias.double(), padding=1)
    mag = F.conv2d(rs.abs(), w.double().abs(), bias.double().abs(), padding=1)
    B = segs.shape[0]
    y = y.permute(0, 2, 3, 1).reshape(B * out_size * out_size, 3)
    mag = mag.permute(0, 2, 3, 1).reshape(B * out_size * out_size, 3)
    n = Cin * out_size * out_size
    ss = rs.sum(dim=(1, 2, 3))
    return (y, 2 * U[out_dtype] * y.abs() + 2 * 9 * Cin * E32 * mag + ETA[out_dtype], ss,
            2 * n * E32 * rs.abs().sum(dim=(1, 2, 3)))


def seg_tokens64(feat, null_pos, pos, seg_sum, batch, pixels, tokens):
    """feat NHWC [B P, C] -> rows [B T, C P / T]: the NCHW map's reshape(B, -1, T).permute(0, 2, 1) + pos where the
    image has a mask (seg_sum > 0), null_pos where it has none."""
    C = feat.shape[-1]
    f = feat.double().reshape(batch, pixels, C).permute(0, 2, 1).reshape(batch, -1, tokens).permute(0, 2, 1)
    y = f + pos.double()
    has = (seg_sum.double() > 0)[:, None, None]
    return torch.where(has, y, null_pos.double().expand_as(y)).reshape(batch * tokens, -1)


# exact layout ops: the expected tensor itself
def im2col_s2_ref(x, batch, h, w, pad01=False):
    C = x.shape[-1]
    xn = x.reshape(batch, h, w, C).permute(0, 3, 1, 2).double()
    if pad01:
        cols = F.unfold(F.pad(xn, (0, 1, 0, 1)), 3, padding=0, stride=2)
    else:
        cols = F.unfold(xn, 3, padding=1, stride=2)
    L = cols.shape[-1]
    return cols.reshape(batch, C, 9, L).permute(0, 3, 2, 1).reshape(batch * L, 9 * C).to(x.dtype)


def upsample_nearest2x_ref(x, batch, h, w):
    C = x.shape[-1]
    return x.reshape(batch, h, w, C).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1, C)


def patchify_ref(x, batch, h, w, c, p):
    return x.reshape(batch, h // p, p, w // p, p, c).permute(0, 1, 3, 2, 4, 5).reshape(batch * (h // p) * (w // p),
                                                                                        p * p * c)


def nchw_to_nhwc_ref(x, c_pad, out_dtype):
    B, C, H, W = x.shape
    out = torch.zeros((B * H * W, c_pad), dtype=out_dtype, device=x.device)
    out[:, :C] = x.permute(0, 2, 3, 1).reshape(-1, C).to(out_dtype)
    return out


# --------------------------------------------------------------------------------------------
# sampling updates (the others reuse cases_ddim / cases_dpm / cases_img2img / cases_inpaint)
# --------------------------------------------------------------------------------------------
def plms_update64(x, e_c, e_u, gs, olds, coefs, a_t, a_prev, sqrt_one_minus_at):
    """(e64, x_prev64) of ops.plms_update (test_kernels_gpu.py::test_plms_update_and_mean)."""
    e = e_c.double() if e_u is None else e_u.double() + gs * (e_c.double() - e_u.double())
    ep = coefs[0] * e
    for c, o in zip(coefs[1:], olds):
        ep = ep + c * o.double()
    pred = (x.double() - sqrt_one_minus_at * ep) / math.sqrt(a_t)
    return e, math.sqrt(a_prev) * pred + math.sqrt(1 - a_prev) * ep


def latent_mean64(xs):
    return sum(x.double() for x in xs) / len(xs)


def ratio(got, y64, bound) -> float:
    """Worst err / bound; inf for a non-finite output."""
    g = got.double().reshape(y64.shape)
    if not torch.isfinite(g).all():
        return math.inf
    return ((g - y64).abs() / bound).max().item()
