"""Transformer operators of the UNet, same class names / constructor and forward signatures /
state_dict keys as the reference's ldm/modules/attention.py, with the arithmetic in
libidiff_b200.so (wgmma GEMM + flash attention + LayerNorm/GroupNorm kernels).

Internal convention: token-major fp16 activations `[B*N, C]` (== NHWC), carried between the
`_fwd` methods without any NCHW<->(B,HW,C) rearrange (attention.py:369,376 disappear).
The public `forward` methods keep the reference layouts and are used for module-level parity.

LayerNorm never runs as its own pass on the visual stream: LN(x) W^T + b = rstd (x W'^T - mean colsum(W'))
+ (W beta + b) with W' = W * gamma, so the GEMM that consumes a LayerNorm reads the un-normalised stream
with gamma-folded weights and applies (mean, rstd) per row in its epilogue; the row statistics are partial
sums written by the epilogue of the GEMM that produced the stream (ops.RowStats, idiff_gemm_args.ln_*).
The `ln=` arguments below carry (RowStats, ops.LnFold); parents own the fold because the LayerNorm
parameters live in the parent block (attention.py:294-295, 320-322).
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ... import ops
from ...packing import pack_conv1x1, pack_geglu
from ._base import PackedModule, f32, nchw_to_nhwc16, nhwc16_to_nchw, to_tokens, w16
from .diffusionmodules.util import zero_module


def exists(val):
    return val is not None


def default(val, d):
    if exists(val):
        return val
    return d() if callable(d) else d


# --------------------------------------------------------------------------------------------
# feed-forward
# --------------------------------------------------------------------------------------------
class GEGLU(PackedModule):
    """attention.py:36-43: proj -> chunk(2) -> x * gelu(gate) (exact erf GELU), fused into the
    GEMM epilogue (value/gate rows interleaved per 64 at pack time)."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def _pack(self):
        wp, bp = pack_geglu(w16(self.proj.weight), f32(self.proj.bias))
        return {"w": wp, "b": bp}

    def _fwd(self, x16: torch.Tensor, ln=None) -> torch.Tensor:
        if ln is not None:  # (RowStats of x16, LnFold of this projection): x16 is the un-normalised stream
            st, f = ln
            return ops.gemm(x16, f.w, f.bias, geglu=True, ln=(st, f.colsum, f.eps))
        p = self.pk()
        return ops.gemm(x16, p["w"], p["b"], geglu=True)

    def fold(self, norm: nn.LayerNorm) -> "ops.LnFold":
        return ops.fold_layernorm(self.proj.weight, self.proj.bias, norm.weight, norm.bias, norm.eps, pack=pack_geglu)

    def forward(self, x):
        x16, B, N = to_tokens(x)
        return self._fwd(x16).view(B, N, -1).to(x.dtype)


class FeedForward(PackedModule):
    """attention.py:46-63 with glu=True (the only configuration the UNet builds)."""

    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.):
        super().__init__()
        inner_dim = int(dim * mult)
        dim_out = default(dim_out, dim)
        if not glu:
            raise NotImplementedError("FeedForward(glu=False) is not on the InstanceDiffusion path")
        self.net = nn.Sequential(GEGLU(dim, inner_dim), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out))

    def _pack(self):
        return {"w2": w16(self.net[2].weight), "b2": f32(self.net[2].bias)}

    def _fwd(self, x16, residual=None, gate=1.0, out=None, ln=None, want_stats=False, gate_rows=None, rows_per_batch=0):
        """x16: LayerNorm-ed input (or, with ln=(RowStats, LnFold), the stream itself).  Returns residual +
        gate * FF(x16) (or FF(x16) without residual); with want_stats also the RowStats of the result.
        gate_rows: fp32 per-image factor of the gate (images of rows_per_batch rows), see ops.gemm."""
        p = self.pk()
        h = self.net[0]._fwd(x16, ln=ln)
        return ops.gemm(h, p["w2"], p["b2"], residual=residual, gate=gate, out=out, want_stats=want_stats,
                        gate_rows=gate_rows, rows_per_batch=rows_per_batch)

    def forward(self, x):
        x16, B, N = to_tokens(x)
        return self._fwd(x16).view(B, N, -1).to(x.dtype)


# --------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------
class CrossAttention(PackedModule):
    """attention.py:98-157.  K/V of the 77 text tokens are step-invariant: `project_kv` is hoisted
    by the UNet (once per prompt), `_fwd` then needs only the Q projection."""

    def __init__(self, query_dim, key_dim, value_dim, heads=8, dim_head=64, dropout=0, efficient_attention=False):
        super().__init__()
        inner_dim = dim_head * heads
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.efficient_attention = efficient_attention
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(key_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(value_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))

    def _pack(self):
        return {
            "wkv": torch.cat([w16(self.to_k.weight), w16(self.to_v.weight)], 0).contiguous(),
            "wo": w16(self.to_out[0].weight),
            "bo": f32(self.to_out[0].bias),
        }

    def fold_q(self, norm: nn.LayerNorm) -> "ops.LnFold":
        return ops.fold_layernorm(self.to_q.weight, None, norm.weight, norm.bias, norm.eps)

    def project_kv(self, ctx16: torch.Tensor) -> torch.Tensor:
        """ctx16 fp16 [B*M, key_dim] -> [B*M, 2*inner] = [K | V]."""
        return ops.gemm(ctx16, self.pk()["wkv"])

    def _fwd(self, x16, kv, B, N, M, residual=None, out=None, ln=None, want_stats=False):
        p = self.pk()
        C = self.heads * self.dim_head
        if ln is not None:
            st, f = ln
            q = ops.gemm(x16, f.w, f.bias, ln=(st, f.colsum, f.eps))
        else:
            q = ops.gemm(x16, self.lazy("wq", lambda: w16(self.to_q.weight)))
        a = ops.attention(q, kv[:, :C], kv[:, C:2 * C], batch=B, heads=self.heads, head_dim=self.dim_head,
                          nq=N, n0=M, scale=self.scale)
        return ops.gemm(a, p["wo"], p["bo"], residual=residual, out=out, want_stats=want_stats)

    def forward(self, x, key, value, mask=None):
        if mask is not None:
            raise NotImplementedError("CrossAttention mask is unused on the shipped sampling path")
        if key is not value:
            raise NotImplementedError("CrossAttention expects key is value (attention.py:336 passes context twice)")
        x16, B, N = to_tokens(x)
        c16, _, M = to_tokens(key)
        return self._fwd(x16, self.project_kv(c16), B, N, M).view(B, N, -1).to(x.dtype)


class SelfAttention(PackedModule):
    """attention.py:160-282 (efficient_attention path; the instance attention-mask builder at
    :187-255 is dead under every shipped config, SURVEY.md section 5)."""

    def __init__(self, query_dim, heads=8, dim_head=64, dropout=0., efficient_attention=False):
        super().__init__()
        inner_dim = dim_head * heads
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.efficient_attention = efficient_attention
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))

    def _pack(self):
        return {"wo": w16(self.to_out[0].weight), "bo": f32(self.to_out[0].bias)}

    def _wqkv(self):
        return torch.cat([w16(self.to_q.weight), w16(self.to_k.weight), w16(self.to_v.weight)], 0).contiguous()

    def fold_qkv(self, norm: nn.LayerNorm) -> "ops.LnFold":
        w = torch.cat([self.to_q.weight.detach(), self.to_k.weight.detach(), self.to_v.weight.detach()], 0)
        return ops.fold_layernorm(w, None, norm.weight, norm.bias, norm.eps)

    def project_kv(self, x16: torch.Tensor) -> torch.Tensor:
        wkv = self.lazy("wkv", lambda: torch.cat([w16(self.to_k.weight), w16(self.to_v.weight)], 0).contiguous())
        return ops.gemm(x16, wkv)

    def _fwd(self, x16, B, N, residual=None, gate=1.0, extra_kv=None, n_extra=0, extra_batch=0, out=None, ln=None,
             want_stats=False, mask=None, gate_rows=None):
        """x16: normalised tokens [B*N, C] -- or, with ln=(RowStats, LnFold), the un-normalised stream.
        extra_kv: [Be*n_extra, 2C] additional keys/values (the object tokens of the gated block).
        gate_rows: fp32 [B] per-image factor of the residual gate (ops.gemm)."""
        p = self.pk()
        C = self.heads * self.dim_head
        if ln is not None:
            st, f = ln
            qkv = ops.gemm(x16, f.w, f.bias, ln=(st, f.colsum, f.eps))
        else:
            qkv = ops.gemm(x16, self.lazy("wqkv", self._wqkv))
        kw = {}
        if extra_kv is not None:
            kw = dict(k1=extra_kv[:, :C], v1=extra_kv[:, C:2 * C], n1=n_extra, kv1_batch=extra_batch)
        if mask is not None:  # instance-isolation mask words (attention.py:187-255; ops.attmask_words)
            kw["mask"] = mask
        a = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], batch=B, heads=self.heads,
                          head_dim=self.dim_head, nq=N, n0=N, scale=self.scale, **kw)
        return ops.gemm(a, p["wo"], p["bo"], residual=residual, gate=gate, out=out, want_stats=want_stats,
                        gate_rows=gate_rows, rows_per_batch=N if gate_rows is not None else 0)

    def forward(self, x, grounding_input=None, drop_box_mask=False):
        x16, B, N = to_tokens(x)
        return self._fwd(x16, B, N).view(B, N, -1).to(x.dtype)


class GatedSelfAttentionDense(PackedModule):
    """attention.py:285-311, restructured (exact in real arithmetic, SURVEY.md section 7):
    LayerNorm is per token, so norm1(cat[x, objs']) = cat[norm1 x, norm1 objs']; queries, the
    out-projection and the softmax rows are computed only for the N visual tokens (the only rows
    the reference keeps, :308) while the 184 object rows contribute keys/values -- computed once
    per sample by `project_objs` and reused for all steps."""

    def __init__(self, query_dim, context_dim, n_heads, d_head, efficient_attention=False):
        super().__init__()
        self.linear = nn.Linear(context_dim, query_dim)
        self.attn = SelfAttention(query_dim=query_dim, heads=n_heads, dim_head=d_head,
                                  efficient_attention=efficient_attention)
        self.ff = FeedForward(query_dim, glu=True)
        self.norm1 = nn.LayerNorm(query_dim)
        self.norm2 = nn.LayerNorm(query_dim)
        self.register_parameter('alpha_attn', nn.Parameter(torch.tensor(0.)))
        self.register_parameter('alpha_dense', nn.Parameter(torch.tensor(0.)))
        # set per step by utils.model.set_alpha_scale (1 for the first alpha*S steps, then 0)
        self.scale = 1

    def _pack(self):
        return {
            "wl": w16(self.linear.weight), "bl": f32(self.linear.bias),
            "g1": f32(self.norm1.weight), "b1": f32(self.norm1.bias),  # objects: standalone LayerNorm (hoisted)
            "qkv": self.attn.fold_qkv(self.norm1),
            "ff": self.ff.net[0].fold(self.norm2),
            "tanh_attn": math.tanh(float(self.alpha_attn.detach().float().cpu())),
            "tanh_dense": math.tanh(float(self.alpha_dense.detach().float().cpu())),
        }

    def project_objs(self, objs16: torch.Tensor) -> torch.Tensor:
        """objs16 fp16 [Bo*184, context_dim] -> K|V rows [Bo*184, 2C] = [Wk;Wv] norm1(linear(objs))."""
        p = self.pk()
        o = ops.gemm(objs16, p["wl"], p["bl"])
        o = ops.layernorm(o, p["g1"], p["b1"], self.norm1.eps)
        return self.attn.project_kv(o)

    def mask_applies(self, N: int, n_obj: int, n_inst: int) -> bool:
        """attention.py:190-199: the instance-isolation mask is built only without `efficient_attention` and only
        where the visual tokens are the 64x64 grid (N + n_obj - 4 * n_inst - 64 == 64 * 64)."""
        return (not self.attn.efficient_attention) and N + n_obj - 4 * n_inst - 64 == 64 * 64

    def _fwd(self, x16, stats, B, N, obj_kv, n_obj, obj_batch, mask=None, scale=None):
        """In-place on x16 (the residual stream; `stats` = its RowStats).  Returns (x16, stats).  Identity
        when scale == 0 (the alpha=0 steps).  mask: (mask_q, mask_k) words of ops.attmask_words or None.
        scale: None (this module's `.scale`), a float, or an fp32 [B] tensor of per-image scales (batched requests
        at different alpha steps: the gates become tanh(alpha) * scale[b]; rows with scale 0 pass unchanged)."""
        if scale is None:
            scale = self.scale
        rows = scale if isinstance(scale, torch.Tensor) else None
        if rows is None and scale == 0:
            return x16, stats
        p = self.pk()
        s = 1.0 if rows is not None else float(scale)
        x16, stats = self.attn._fwd(x16, B, N, residual=x16, gate=s * p["tanh_attn"],
                                    extra_kv=obj_kv, n_extra=n_obj, extra_batch=obj_batch, out=x16,
                                    ln=(stats, p["qkv"]), want_stats=True, mask=mask, gate_rows=rows)
        return self.ff._fwd(x16, residual=x16, gate=s * p["tanh_dense"], out=x16,
                            ln=(stats, p["ff"]), want_stats=True, gate_rows=rows, rows_per_batch=N if rows is not None else 0)

    def forward(self, x, objs, grounding_input=None, drop_box_mask=False):
        x16, B, N = to_tokens(x)
        o16, Bo, n_obj = to_tokens(objs)
        x16 = x16.clone()
        mask = attention_mask_words(self, grounding_input, drop_box_mask, B, N, n_obj)
        y, _ = self._fwd(x16, ops.row_stats(x16), B, N, self.project_objs(o16), n_obj, Bo, mask=mask)
        return y.view(B, N, -1).to(x.dtype)


def attention_mask_words(fuser: "GatedSelfAttentionDense", grounding_input, drop_box_mask, B, N, n_obj):
    """attention.py:187-255 as the bit words of ops.attmask_words, or None when the reference builds no mask:
    no `att_masks` in the grounding input, `efficient_attention`, another resolution than 64x64, all-zero masks
    or dropped boxes (:201).  One device->host read of the mask sum (the reference does the same, :201)."""
    if grounding_input is None or "att_masks" not in grounding_input:
        return None
    att = grounding_input["att_masks"]
    n_inst = att.shape[1]
    if not fuser.mask_applies(N, n_obj, n_inst):
        return None
    if drop_box_mask or not bool((att.sum() > 0).item()):
        return None
    active = torch.ones((B,), dtype=torch.int32, device=att.device)
    return ops.attmask_words(att.float().expand(B, -1, -1, -1) if att.shape[0] != B else att.float(), active,
                             tail=n_obj - 4 * n_inst)


class BasicTransformerBlock(PackedModule):
    """attention.py:314-338: x = attn1(LN x)+x; x = fuser(x, objs); x = attn2(LN x, ctx)+x;
    x = ff(LN x)+x.  All residual adds are GEMM epilogues writing the stream in place."""

    def __init__(self, query_dim, key_dim, value_dim, n_heads, d_head, fuser_type, use_checkpoint=True,
                 efficient_attention=False):
        super().__init__()
        self.attn1 = SelfAttention(query_dim=query_dim, heads=n_heads, dim_head=d_head,
                                   efficient_attention=efficient_attention)
        self.ff = FeedForward(query_dim, glu=True)
        self.attn2 = CrossAttention(query_dim=query_dim, key_dim=key_dim, value_dim=value_dim, heads=n_heads,
                                    dim_head=d_head, efficient_attention=efficient_attention)
        self.norm1 = nn.LayerNorm(query_dim)
        self.norm2 = nn.LayerNorm(query_dim)
        self.norm3 = nn.LayerNorm(query_dim)
        self.use_checkpoint = use_checkpoint
        self.fuser = GatedSelfAttentionDense(query_dim, key_dim, n_heads, d_head,
                                             efficient_attention=efficient_attention)

    def _pack(self):
        return {
            "qkv1": self.attn1.fold_qkv(self.norm1),
            "q2": self.attn2.fold_q(self.norm2),
            "ff": self.ff.net[0].fold(self.norm3),
        }

    def _fwd(self, x16, stats, B, N, ctx_kv, M, obj_kv, n_obj, obj_batch, mask=None, fuser_scale=None):
        """x16: the residual stream (updated in place), stats: its RowStats (from the GEMM that wrote it).
        mask: instance-isolation mask words for the fuser (64x64 level, efficient_attention=False) or None.
        fuser_scale: overrides the fuser's `.scale` (GatedSelfAttentionDense._fwd `scale`)."""
        p = self.pk()
        x16, stats = self.attn1._fwd(x16, B, N, residual=x16, out=x16, ln=(stats, p["qkv1"]), want_stats=True)
        x16, stats = self.fuser._fwd(x16, stats, B, N, obj_kv, n_obj, obj_batch, mask=mask, scale=fuser_scale)
        x16, stats = self.attn2._fwd(x16, ctx_kv, B, N, M, residual=x16, out=x16, ln=(stats, p["q2"]), want_stats=True)
        return self.ff._fwd(x16, residual=x16, out=x16, ln=(stats, p["ff"]))

    def forward(self, x, context, objs, grounding_input=None, drop_box_mask=False):
        return self._forward(x, context, objs, grounding_input, drop_box_mask=drop_box_mask)

    def _forward(self, x, context, objs, grounding_input=None, drop_box_mask=False):
        x16, B, N = to_tokens(x)
        c16, _, M = to_tokens(context)
        o16, Bo, n_obj = to_tokens(objs)
        obj_kv = self.fuser.project_objs(o16) if self.fuser.scale != 0 else None
        x16 = x16.clone()
        mask = attention_mask_words(self.fuser, grounding_input, drop_box_mask, B, N, n_obj)
        y = self._fwd(x16, ops.row_stats(x16), B, N, self.attn2.project_kv(c16), M, obj_kv, n_obj, Bo, mask=mask)
        return y.view(B, N, -1).to(x.dtype)


def Normalize(in_channels):
    return torch.nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class SpatialTransformer(PackedModule):
    """attention.py:341-379: GroupNorm(eps 1e-6) -> 1x1 conv -> blocks -> 1x1 conv -> + x_in.
    With NHWC activations the two rearranges are no-ops and the 1x1 convs are plain GEMMs; the
    final residual is the proj_out GEMM's epilogue."""

    def __init__(self, in_channels, key_dim, value_dim, n_heads, d_head, depth=1, fuser_type=None,
                 use_checkpoint=True, efficient_attention=False):
        super().__init__()
        self.in_channels = in_channels
        query_dim = n_heads * d_head
        self.norm = Normalize(in_channels)
        self.proj_in = nn.Conv2d(in_channels, query_dim, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(query_dim, key_dim, value_dim, n_heads, d_head, fuser_type,
                                  use_checkpoint=use_checkpoint, efficient_attention=efficient_attention)
            for _ in range(depth)])
        self.proj_out = zero_module(nn.Conv2d(query_dim, in_channels, kernel_size=1, stride=1, padding=0))

    def _pack(self):
        return {
            "gn_g": f32(self.norm.weight), "gn_b": f32(self.norm.bias),
            "w_in": pack_conv1x1(w16(self.proj_in.weight)), "b_in": f32(self.proj_in.bias),
            "w_out": pack_conv1x1(w16(self.proj_out.weight)), "b_out": f32(self.proj_out.bias),
        }

    def _fwd(self, x16, B, H, W, ctx_kvs, M, obj_kvs, n_obj, obj_batch, mask=None, fuser_scale=None):
        """x16 fp16 [B*H*W, C].  ctx_kvs / obj_kvs: one entry per transformer block.  mask, fuser_scale: see
        BasicTransformerBlock."""
        p = self.pk()
        n = ops.groupnorm(x16, p["gn_g"], p["gn_b"], batch=B, hw=H * W, groups=32, eps=self.norm.eps, silu=False)
        t, stats = ops.gemm(n, p["w_in"], p["b_in"], want_stats=True)
        for i, blk in enumerate(self.transformer_blocks):
            if i > 0:  # (depth > 1: the previous block's FF out-projection did not keep statistics)
                stats = ops.row_stats(t)
            t = blk._fwd(t, stats, B, H * W, ctx_kvs[i], M, obj_kvs[i] if obj_kvs is not None else None, n_obj, obj_batch,
                         mask=mask if H * W == 64 * 64 else None, fuser_scale=fuser_scale)
        return ops.gemm(t, p["w_out"], p["b_out"], residual=x16)

    def forward(self, x, context, objs, grounding_input=None, drop_box_mask=False):
        x16, B, H, W = nchw_to_nhwc16(x)
        c16, _, M = to_tokens(context)
        o16, Bo, n_obj = to_tokens(objs)
        ctx_kvs = [blk.attn2.project_kv(c16) for blk in self.transformer_blocks]
        obj_kvs = [blk.fuser.project_objs(o16) if blk.fuser.scale != 0 else None for blk in self.transformer_blocks]
        mask = attention_mask_words(self.transformer_blocks[0].fuser, grounding_input, drop_box_mask, B, H * W, n_obj)
        y = self._fwd(x16, B, H, W, ctx_kvs, M, obj_kvs, n_obj, Bo, mask=mask)
        return nhwc16_to_nchw(y, B, H, W, x.dtype)
