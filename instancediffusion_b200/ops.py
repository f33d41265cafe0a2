"""Thin torch-tensor front end of the C ABI (include/idiff_b200.h).

torch is used only for device memory and the current stream; all arithmetic happens in
libidiff_b200.so.  Every function enqueues on torch's current CUDA stream and returns the output
tensor without synchronising.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import AttnArgs, GemmArgs, check

# 16-bit storage type of activations and packed weights: process-wide, fp16 (the reference's autocast type,
# inference.py:94) unless set_storage_dtype(torch.bfloat16) selects the bf16 build of the library (BASELINE
# config 3).  Every wrapper below checks its 16-bit operands against it, so tensors of the other type fail
# loudly instead of being reinterpreted.
HALF = torch.float16
STORAGE_EPOCH = 0  # bumped on every switch: weight packs and hoisted tensors built before it are stale
_KINDS = {torch.float16: "f16", torch.bfloat16: "bf16"}


def set_storage_dtype(dtype: torch.dtype) -> None:
    """Select the 16-bit storage type (torch.float16 or torch.bfloat16) for everything created afterwards.
    Modules re-pack their weights and the UNet drops its hoisted tensors / captured graphs on next use."""
    global HALF, STORAGE_EPOCH
    if dtype not in _KINDS:
        raise _lib.IdiffError(f"storage dtype must be torch.float16 or torch.bfloat16, got {dtype}")
    if dtype != HALF:
        _lib.set_storage(_KINDS[dtype])
        HALF = dtype
        STORAGE_EPOCH += 1


def storage_dtype() -> torch.dtype:
    return HALF


class storage:
    """Context manager: `with ops.storage(torch.bfloat16): ...`."""

    def __init__(self, dtype: torch.dtype):
        self.dtype = dtype

    def __enter__(self):
        self.prev = HALF
        set_storage_dtype(self.dtype)
        return self

    def __exit__(self, *exc):
        set_storage_dtype(self.prev)
        return False


# Optional per-launch timing (bench.py's roofline pass): when PROFILE is a list, every wrapper
# brackets its launch with CUDA events on the launching stream and appends
# (kind, algorithmic_flops, algorithmic_bytes, start_event, end_event).
PROFILE = None


def _launch(kind: str, flops: float, nbytes: float, fn):
    if PROFILE is None:
        return fn()
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    s.record()
    rc = fn()
    e.record()
    PROFILE.append((kind, flops, nbytes, s, e))
    return rc


_GEMM_WS = {}


_WS_SCOPE = None  # when set (capture_workspace()), every GEMM uses this key's buffer


def _ws_buffer(key, device: torch.device) -> torch.Tensor:
    buf = _GEMM_WS.get(key)
    if buf is None:
        n = int(_lib.load().idiff_gemm_workspace_bytes())
        buf = torch.zeros(n, dtype=torch.uint8, device=device)  # flags must start at zero
        _GEMM_WS[key] = buf
    return buf


def _gemm_workspace(device: torch.device):
    """Stream-K scratch (flags + fp32 partial tiles) for this call, passed in idiff_gemm_args.workspace:
    one buffer per (device, stream), so GEMMs in flight on different streams never share flags.  Work
    recorded into CUDA graphs uses one per-device buffer (`capture_workspace`): replays are ordered on
    the replaying stream.  Never allocates during stream capture (falls back to data-parallel GEMMs)."""
    if _WS_SCOPE is not None:
        key = (device.index, _WS_SCOPE)
    else:
        key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _GEMM_WS.get(key)
    if buf is None:
        if torch.cuda.is_current_stream_capturing():
            return None, 0
        buf = _ws_buffer(key, device)
    return buf.data_ptr(), buf.numel()


class capture_workspace:
    """Context: GEMMs issued inside (graph warm-up and capture) use the device's graph scratch buffer,
    allocated on entry -- i.e. outside the capture."""

    def __init__(self, device: torch.device):
        self.device = device

    def __enter__(self):
        global _WS_SCOPE
        _ws_buffer((self.device.index, "graph"), self.device)
        self._prev, _WS_SCOPE = _WS_SCOPE, "graph"
        return self

    def __exit__(self, *exc):
        global _WS_SCOPE
        _WS_SCOPE = self._prev
        return False


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise _lib.IdiffError(f"{name} must be a CUDA tensor (no CPU fallback exists)")
    if t.dtype != dtype:
        raise _lib.IdiffError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1:
        raise _lib.IdiffError(f"{name} must be contiguous in its last dimension")


class RowStats:
    """Per-row partial (sum, sum of squares) of a token matrix, fp32 [slots, rows, 2]: what a producer GEMM's
    epilogue (or row_stats) leaves for the folded LayerNorm of the next GEMM (idiff_gemm_args.ln_*)."""
    __slots__ = ("t", "slots")

    def __init__(self, t: torch.Tensor, slots: int):
        self.t, self.slots = t, slots


class LnFold:
    """LayerNorm folded into the GEMM that consumes its output: w = fp16(W * gamma) (already in the layout
    the GEMM wants), colsum[n] = sum_k w[n, k] (fp32), bias = W beta + b (fp32), eps."""
    __slots__ = ("w", "bias", "colsum", "eps")

    def __init__(self, w, bias, colsum, eps):
        self.w, self.bias, self.colsum, self.eps = w, bias, colsum, float(eps)


def fold_layernorm(weight: torch.Tensor, bias: Optional[torch.Tensor], ln_weight: torch.Tensor, ln_bias: torch.Tensor,
                   eps: float, pack=None) -> LnFold:
    """LN(x) W^T + b = rstd (x W'^T - mean colsum(W')) + (W beta + b), W' = W * gamma (fp32 masters in).
    `pack(w16, b32) -> (w16, b32)` re-lays rows out (GEGLU interleave) before the column sums are taken."""
    W = weight.detach().float()
    g = ln_weight.detach().float()
    beta = ln_bias.detach().float()
    w16 = (W * g[None, :]).to(HALF).contiguous()
    b = W @ beta
    if bias is not None:
        b = b + bias.detach().float()
    b = b.contiguous()
    if pack is not None:
        w16, b = pack(w16, b)
    return LnFold(w16, b, w16.float().sum(dim=1).contiguous(), eps)


def row_stats(x: torch.Tensor) -> RowStats:
    """One-slot row statistics of an fp16 [rows, C] matrix (entry of the folded LayerNorm when the stream was
    not written by a GEMM of this library)."""
    lib = _lib.load()
    _req(x, HALF, "x")
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        raise _lib.IdiffError("row_stats input must be contiguous")
    st = torch.empty((1, x2.shape[0], 2), dtype=torch.float32, device=x.device)
    check(_launch("row_stats", 0.0, 2.0 * x2.numel(), lambda: lib.idiff_row_stats(
        x2.data_ptr(), st.data_ptr(), x2.shape[0], x2.shape[1], _stream())), "idiff_row_stats")
    return RowStats(st, 1)


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
         out: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         gate: float = 1.0, rowadd: Optional[torch.Tensor] = None, rows_per_batch: int = 0,
         geglu: bool = False, silu: bool = False, gelu: bool = False,
         conv: Optional[Tuple[int, int, int, int]] = None,
         out_nchw: Optional[torch.Tensor] = None,
         ln: Optional[Tuple["RowStats", torch.Tensor, float]] = None, want_stats: bool = False,
         gate_rows: Optional[torch.Tensor] = None):
    """out = epilogue(a @ w.T).  a: fp16 [M,K] (or NHWC [B,H,W,Cin] flattened with conv=(B,H,W,Cin));
    w: fp16 [N,K].  See idiff_gemm in include/idiff_b200.h.
    ln = (RowStats of a's rows, colsum, eps): a is the un-normalised stream and w / bias are LayerNorm-folded
    (fold_layernorm).  want_stats: also return the RowStats of the output rows -> (out, stats).
    gate_rows: fp32 [batch entries] (entry = row // rows_per_batch, conv: the image) multiplying `gate` per
    entry: out = residual + gate * gate_rows[b] * (...).  Needs `residual`."""
    lib = _lib.load()
    _req(a, HALF, "a")
    _req(w, HALF, "w")
    N, K = w.shape
    if conv is not None:
        B, H, Wd, Cin = conv
        M = B * H * Wd
        a2 = a.reshape(M, Cin)
        lda = Cin
        if not a2.is_contiguous():
            raise _lib.IdiffError("conv activation must be contiguous NHWC")
    else:
        a2 = a.reshape(-1, a.shape[-1])
        M = a2.shape[0]
        lda = a2.stride(0)
        if a2.shape[1] != K:
            raise _lib.IdiffError(f"gemm: K mismatch a[{a2.shape}] w[{w.shape}]")
    n_out = N // 2 if geglu else N
    flags = (1 if geglu else 0) | (2 if silu else 0) | (8 if gelu else 0)
    args = GemmArgs()
    if out_nchw is not None:
        _req(out_nchw, torch.float32, "out_nchw")
        flags |= 4
        args.out = out_nchw.data_ptr()
        args.ldo = 0
        result = out_nchw
    else:
        if out is None:
            out = torch.empty((M, n_out), dtype=HALF, device=a.device)
        _req(out, HALF, "out")
        args.out = out.data_ptr()
        args.ldo = out.stride(0) if out.dim() == 2 else n_out
        result = out
    args.a = a2.data_ptr()
    args.w = w.data_ptr()
    if bias is not None:
        _req(bias, torch.float32, "bias")
    args.bias = _ptr(bias)
    if rowadd is not None:
        _req(rowadd, HALF, "rowadd")
        args.ldra = rowadd.stride(0)
    args.rowadd = _ptr(rowadd)
    if residual is not None:
        _req(residual, HALF, "residual")
        args.ldr = residual.stride(0)
    args.residual = _ptr(residual)
    args.gate = float(gate)
    if gate_rows is not None:
        _req(gate_rows, torch.float32, "gate_rows")
        entries = conv[0] if conv is not None else -(-M // (rows_per_batch if rows_per_batch > 0 else M))
        if residual is None or not gate_rows.is_contiguous() or gate_rows.numel() < entries:
            raise _lib.IdiffError(f"gemm: gate_rows needs a residual and {entries} contiguous entries "
                                  f"(got {tuple(gate_rows.shape)})")
        args.gate_b = gate_rows.data_ptr()
    args.workspace, args.workspace_bytes = _gemm_workspace(a.device)
    args.M, args.N, args.K = M, N, K
    args.lda, args.ldw = lda, w.stride(0)
    args.rows_per_batch = rows_per_batch
    args.flags = flags
    if conv is not None:
        args.conv_b, args.conv_h, args.conv_w, args.conv_cin = conv
    if ln is not None:
        st, colsum, eps = ln
        _req(colsum, torch.float32, "ln colsum")
        if st.t.shape[1] != M or colsum.numel() != N:
            raise _lib.IdiffError(f"gemm: LayerNorm fold shape mismatch (stats rows {st.t.shape[1]} vs M {M}, "
                                  f"colsum {colsum.numel()} vs N {N})")
        args.ln_stats_in = st.t.data_ptr()
        args.ln_colsum = colsum.data_ptr()
        args.ln_slots_in = st.slots
        args.ln_eps = float(eps)
    stats = None
    if want_stats:
        slots = lib.idiff_gemm_ln_slots(C.byref(args))
        if slots <= 0:
            check(-1, "idiff_gemm_ln_slots")
        stats = RowStats(torch.empty((slots, M, 2), dtype=torch.float32, device=a.device), slots)
        args.ln_stats_out = stats.t.data_ptr()
    kind = "conv3x3" if conv is not None else ("gemm_geglu" if geglu else "gemm")
    nbytes = 2.0 * (M * K / (9 if conv is not None else 1) + N * K + M * n_out)
    check(_launch(kind, 2.0 * M * N * K, nbytes, lambda: lib.idiff_gemm(C.byref(args), _stream())), "idiff_gemm")
    return (result, stats) if want_stats else result


def attention(q: torch.Tensor, k0: torch.Tensor, v0: torch.Tensor, *, batch: int, heads: int,
              head_dim: int, nq: int, n0: int, scale: float,
              k1: Optional[torch.Tensor] = None, v1: Optional[torch.Tensor] = None, n1: int = 0,
              kv1_batch: int = 0, out: Optional[torch.Tensor] = None,
              mask: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
    """softmax(q k^T scale) v over segment 0 (+ optional segment 1) keys.  q/k/v are 2-D fp16 views
    [batch*rows, >= heads*head_dim] (row stride = .stride(0)); returns fp16 [batch*nq, heads*head_dim].
    mask = (mask_q int32 [batch, nq], mask_k int32 [batch, n0 + n1]) from attmask_words: the instance-isolation
    mask of the gated self-attention (head_dim 40 only)."""
    lib = _lib.load()
    for name, t in (("q", q), ("k0", k0), ("v0", v0)):
        _req(t, HALF, name)
    C_ = heads * head_dim
    if out is None:
        out = torch.empty((batch * nq, C_), dtype=HALF, device=q.device)
    a = AttnArgs()
    a.q, a.k0, a.v0 = q.data_ptr(), k0.data_ptr(), v0.data_ptr()
    a.q_ld, a.k0_ld, a.v0_ld = q.stride(0), k0.stride(0), v0.stride(0)
    if n1 > 0:
        _req(k1, HALF, "k1")
        _req(v1, HALF, "v1")
        a.k1, a.v1 = k1.data_ptr(), v1.data_ptr()
        a.k1_ld, a.v1_ld = k1.stride(0), v1.stride(0)
    a.out = out.data_ptr()
    a.out_ld = out.stride(0)
    a.batch, a.heads, a.head_dim = batch, heads, head_dim
    a.nq, a.n0, a.n1 = nq, n0, n1
    a.kv1_batch = kv1_batch if kv1_batch else batch
    a.scale = float(scale)
    if mask is not None:
        mq, mk = mask
        _req(mq, torch.int32, "mask_q")
        _req(mk, torch.int32, "mask_k")
        if tuple(mq.shape) != (batch, nq) or tuple(mk.shape) != (batch, n0 + n1) or not (mq.is_contiguous() and mk.is_contiguous()):
            raise _lib.IdiffError(f"attention: mask shapes {tuple(mq.shape)} / {tuple(mk.shape)} do not match "
                                  f"(batch {batch}, nq {nq}, keys {n0 + n1})")
        a.mask_q, a.mask_k = mq.data_ptr(), mk.data_ptr()
    flops = 4.0 * batch * heads * nq * (n0 + n1) * head_dim
    nbytes = 2.0 * batch * C_ * (2 * nq + 2 * (n0 + n1))
    check(_launch(f"attention_d{head_dim}", flops, nbytes, lambda: lib.idiff_attention(C.byref(a), _stream())),
          "idiff_attention")
    return out


def groupnorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, batch: int, hw: int,
              groups: int = 32, eps: float = 1e-5, silu: bool = False,
              out: Optional[torch.Tensor] = None, stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, HALF, "x")
    Cc = x.shape[-1]
    if out is None:
        out = torch.empty_like(x)
    if stats_ws is None:
        stats_ws = torch.empty(lib.idiff_groupnorm_ws_floats(batch, groups), dtype=torch.float32, device=x.device)
    check(_launch("groupnorm", 0.0, 4.0 * x.numel(), lambda: lib.idiff_groupnorm(
        x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), stats_ws.data_ptr(), batch, hw, Cc,
        groups, eps, int(silu), _stream())), "idiff_groupnorm")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, HALF, "x")
    x2 = x.reshape(-1, x.shape[-1])
    if not x2.is_contiguous():
        raise _lib.IdiffError("layernorm input must be contiguous")
    if out is None:
        out = torch.empty_like(x2)
    check(_launch("layernorm", 0.0, 4.0 * x2.numel(), lambda: lib.idiff_layernorm(
        x2.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), x2.shape[0], x2.shape[1], eps,
        _stream())), "idiff_layernorm")
    return out


def scaleu_concat(h: torch.Tensor, skip: torch.Tensor, b1: torch.Tensor, s: float, *, batch: int,
                  height: int, width: int, out: Optional[torch.Tensor] = None,
                  coef_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(h, HALF, "h")
    _req(skip, HALF, "skip")
    c1, c2 = h.shape[-1], skip.shape[-1]
    if out is None:
        out = torch.empty((batch * height * width, c1 + c2), dtype=HALF, device=h.device)
    if coef_ws is None:
        coef_ws = torch.empty(lib.idiff_scaleu_ws_floats(batch, c2), dtype=torch.float32, device=h.device)
    check(_launch("scaleu_concat", 0.0, 4.0 * (h.numel() + skip.numel()), lambda: lib.idiff_scaleu_concat(
        h.data_ptr(), skip.data_ptr(), out.data_ptr(), b1.data_ptr(), float(s), coef_ws.data_ptr(), batch, height,
        width, c1, c2, _stream())), "idiff_scaleu_concat")
    return out


def nchw_f32_to_nhwc_f16(x: torch.Tensor, c_pad: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, torch.float32, "x")
    B, Cc, H, W = x.shape
    x = x.contiguous()
    if out is None:
        out = torch.empty((B * H * W, c_pad), dtype=HALF, device=x.device)
    check(lib.idiff_nchw_f32_to_nhwc_f16(x.data_ptr(), out.data_ptr(), B, Cc, H * W, c_pad, _stream()),
          "idiff_nchw_f32_to_nhwc_f16")
    return out


def nhwc_f16_to_nchw_f32(x: torch.Tensor, batch: int, h: int, w: int) -> torch.Tensor:
    lib = _lib.load()
    _req(x, HALF, "x")
    Cc = x.shape[-1]
    out = torch.empty((batch, Cc, h, w), dtype=torch.float32, device=x.device)
    check(lib.idiff_nhwc_f16_to_nchw_f32(x.data_ptr(), out.data_ptr(), batch, Cc, h * w, _stream()),
          "idiff_nhwc_f16_to_nchw_f32")
    return out


def upsample_nearest2x(x: torch.Tensor, batch: int, h: int, w: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, HALF, "x")
    Cc = x.shape[-1]
    if out is None:
        out = torch.empty((batch * 4 * h * w, Cc), dtype=HALF, device=x.device)
    check(lib.idiff_upsample_nearest2x(x.data_ptr(), out.data_ptr(), batch, h, w, Cc, _stream()),
          "idiff_upsample_nearest2x")
    return out


def im2col_s2(x: torch.Tensor, batch: int, h: int, w: int, out: Optional[torch.Tensor] = None,
              pad01: bool = False) -> torch.Tensor:
    """Operand rows of a stride-2 3x3 convolution: padding 1 (UNet Downsample) or, pad01, the first-stage
    encoder's F.pad (0,1,0,1) + padding 0."""
    lib = _lib.load()
    _req(x, HALF, "x")
    Cc = x.shape[-1]
    if out is None:
        out = torch.empty((batch * (h // 2) * (w // 2), 9 * Cc), dtype=HALF, device=x.device)
    fn = lib.idiff_im2col_s2_pad01 if pad01 else lib.idiff_im2col_s2
    check(fn(x.data_ptr(), out.data_ptr(), batch, h, w, Cc, _stream()), "idiff_im2col_s2")
    return out


def fourier_embed(coords: torch.Tensor, masks: torch.Tensor, null_pos: torch.Tensor, out: torch.Tensor, *,
                  text: Optional[torch.Tensor] = None, null_text: Optional[torch.Tensor] = None,
                  mask_mode: int = 0, dropped: bool = False) -> torch.Tensor:
    """coords fp32 [rows, D]; masks fp32 [rows]; out fp16 [rows, text_dim + 32*D] (row stride free)."""
    lib = _lib.load()
    _req(coords, torch.float32, "coords")
    _req(masks, torch.float32, "masks")
    _req(out, HALF, "out")
    rows, D = coords.shape
    text_dim = text.shape[-1] if text is not None else 0
    check(lib.idiff_fourier_embed(coords.data_ptr(), masks.data_ptr(), _ptr(text), _ptr(null_text),
                                  null_pos.data_ptr(), out.data_ptr(), rows, D, text_dim, out.stride(0),
                                  mask_mode, int(dropped), _stream()), "idiff_fourier_embed")
    return out


def timestep_embedding(t: torch.Tensor, dim: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(t, torch.float32, "t")
    B = t.shape[0]
    if out is None:
        out = torch.empty((B, dim), dtype=HALF, device=t.device)
    check(lib.idiff_timestep_embedding(t.data_ptr(), out.data_ptr(), B, dim, _stream()),
          "idiff_timestep_embedding")
    return out


def plms_update(x: torch.Tensor, e_c: torch.Tensor, e_u: Optional[torch.Tensor], gs: float,
                olds, coefs, a_t: float, a_prev: float, sqrt_one_minus_at: float,
                e_out: Optional[torch.Tensor], x_out: torch.Tensor) -> None:
    lib = _lib.load()
    o = list(olds) + [None] * (3 - len(olds))
    c = list(coefs) + [0.0] * (4 - len(coefs))
    check(lib.idiff_plms_update(x.data_ptr(), e_c.data_ptr(), _ptr(e_u), float(gs), _ptr(o[0]), _ptr(o[1]),
                                _ptr(o[2]), c[0], c[1], c[2], c[3], float(a_t), float(a_prev),
                                float(sqrt_one_minus_at), _ptr(e_out), x_out.data_ptr(), x.numel(), _stream()),
          "idiff_plms_update")


def latent_mean(xs, out: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    ptrs = torch.tensor([t.data_ptr() for t in xs], dtype=torch.int64).to(out.device)
    check(lib.idiff_latent_mean(ptrs.data_ptr(), len(xs), out.data_ptr(), out.numel(), _stream()),
          "idiff_latent_mean")
    return out


def conv_in_select(x: torch.Tensor, w0: torch.Tensor, b0: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor,
                   flags: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The UNet input conv with a weight set per image: x fp32 (B, 4, H, W); w0 / w1 16-bit [36, Cout]
    (packing.pack_conv3x3_taps); b0 / b1 fp32 [Cout]; flags int32 (B,) on the device, 0 -> (w0, b0), else
    (w1, b1).  Returns 16-bit NHWC [B*H*W, Cout], the activation the first ResBlock reads."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(flags, torch.int32, "flags")
    B, Cc, H, W = x.shape
    cout = w0.shape[1]
    for name, w, b in (("w0", w0, b0), ("w1", w1, b1)):
        _req(w, HALF, name)
        _req(b, torch.float32, name.replace("w", "b"))
        if tuple(w.shape) != (36, cout) or not w.is_contiguous() or b.numel() != cout:
            raise _lib.IdiffError(f"conv_in_select: {name} {tuple(w.shape)} / bias {tuple(b.shape)} are not [36, {cout}] / [{cout}]")
    if Cc != 4 or flags.numel() != B or not flags.is_contiguous():
        raise _lib.IdiffError(f"conv_in_select: x {tuple(x.shape)} needs 4 channels and flags {B} entries")
    x = x.contiguous()
    if out is None:
        out = torch.empty((B * H * W, cout), dtype=HALF, device=x.device)
    _req(out, HALF, "out")
    check(_launch("conv_in_select", 2.0 * B * H * W * cout * 36, 4.0 * x.numel() + 2.0 * out.numel(),
                  lambda: lib.idiff_conv_in_select(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(),
                                                   flags.data_ptr(), out.data_ptr(), B, H, W, cout, _stream())),
          "idiff_conv_in_select")
    return out


def silu(x: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    _req(x, HALF, "x")
    x = x.contiguous()
    out = torch.empty_like(x)
    check(lib.idiff_silu_f16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "idiff_silu_f16")
    return out


# ------------------------------------------------------------------------------------------------
# ConvNeXt mask encoder pieces (csrc/convnext.cu)
# ------------------------------------------------------------------------------------------------
def patchify(x: torch.Tensor, batch: int, h: int, w: int, c: int, p: int) -> torch.Tensor:
    """NHWC fp16 [B*H*W, C] -> [B*(H/p)*(W/p), p*p*C] (operand of a kernel-p stride-p convolution)."""
    lib = _lib.load()
    _req(x, HALF, "x")
    x = x.contiguous()
    out = torch.empty((batch * (h // p) * (w // p), p * p * c), dtype=HALF, device=x.device)
    check(lib.idiff_patchify(x.data_ptr(), out.data_ptr(), batch, h, w, c, p, _stream()), "idiff_patchify")
    return out


def dwconv7x7(x: torch.Tensor, w49: torch.Tensor, bias: torch.Tensor, batch: int, h: int, w: int) -> torch.Tensor:
    """Depthwise 7x7 padding 3 on NHWC fp16 [B*H*W, C]; w49 fp32 [49, C] tap-major; bias fp32 [C]."""
    lib = _lib.load()
    _req(x, HALF, "x")
    _req(w49, torch.float32, "w49")
    _req(bias, torch.float32, "bias")
    x = x.contiguous()
    c = x.shape[-1]
    out = torch.empty_like(x)
    check(_launch("dwconv7x7", 2.0 * 49 * x.numel(), 4.0 * x.numel(), lambda: lib.idiff_dwconv7x7(
        x.data_ptr(), w49.data_ptr(), bias.data_ptr(), out.data_ptr(), batch, h, w, c, _stream())), "idiff_dwconv7x7")
    return out


def segs_inconv(segs: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, out_size: int):
    """segs fp32 (B, Cin, S, S), any strides (expanded zero views included) -> (NHWC fp16
    [B*out*out, 3] = Conv2d(Cin,3,3,1,1)(nearest-resize(segs, out)), seg_sum fp32 [B])."""
    lib = _lib.load()
    _req(w, torch.float32, "w")
    _req(bias, torch.float32, "bias")
    if not segs.is_cuda or segs.dtype != torch.float32:
        raise _lib.IdiffError("segs must be a CUDA float32 tensor (no CPU fallback exists)")
    B, Cin, S, S2 = segs.shape
    if S != S2:
        raise _lib.IdiffError("segs must be square")
    y = torch.empty((B * out_size * out_size, 3), dtype=HALF, device=segs.device)
    seg_sum = torch.empty((B,), dtype=torch.float32, device=segs.device)
    strides = (C.c_long * 4)(*segs.stride())
    check(lib.idiff_segs_inconv(segs.data_ptr(), strides, w.data_ptr(), bias.data_ptr(), y.data_ptr(),
                                seg_sum.data_ptr(), B, Cin, S, out_size, _stream()), "idiff_segs_inconv")
    return y, seg_sum


def seg_tokens(feat: torch.Tensor, null_pos: torch.Tensor, pos: torch.Tensor, seg_sum: torch.Tensor, batch: int,
               pixels: int, tokens: int) -> torch.Tensor:
    """feat fp16 NHWC [B*P, C] -> MLP input rows fp16 [B*T, C*P/T] (token reinterpretation + null / pos)."""
    lib = _lib.load()
    _req(feat, HALF, "feat")
    _req(null_pos, HALF, "null_pos")
    _req(pos, torch.float32, "pos")
    _req(seg_sum, torch.float32, "seg_sum")
    c = feat.shape[-1]
    out = torch.empty((batch * tokens, c * pixels // tokens), dtype=HALF, device=feat.device)
    check(lib.idiff_seg_tokens(feat.data_ptr(), null_pos.data_ptr(), pos.data_ptr(), seg_sum.data_ptr(),
                               out.data_ptr(), batch, pixels, c, tokens, _stream()), "idiff_seg_tokens")
    return out


# ------------------------------------------------------------------------------------------------
# first-stage decoder pieces (csrc/vae.cu)
# ------------------------------------------------------------------------------------------------
def vae_latent_in(z: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, inv_scale: float) -> torch.Tensor:
    """z fp32 (B, C, H, W) -> fp16 NHWC [B*H*W, 64] = post_quant_conv(z * inv_scale), channels >= C zero."""
    lib = _lib.load()
    _req(z, torch.float32, "z")
    _req(w, torch.float32, "w")
    _req(bias, torch.float32, "bias")
    B, Cc, H, W = z.shape
    z = z.contiguous()
    out = torch.empty((B * H * W, 64), dtype=HALF, device=z.device)
    check(lib.idiff_vae_latent_in(z.data_ptr(), w.data_ptr(), bias.data_ptr(), float(inv_scale), out.data_ptr(), B, Cc,
                                  H * W, _stream()), "idiff_vae_latent_in")
    return out


def softmax_rows_(x: torch.Tensor) -> torch.Tensor:
    """In-place softmax over the last dimension of an fp16 [rows, n] matrix (fp32 arithmetic)."""
    lib = _lib.load()
    _req(x, HALF, "x")
    rows, n = x.shape
    check(_launch("softmax_rows", 0.0, 4.0 * x.numel(), lambda: lib.idiff_softmax_rows(
        x.data_ptr(), rows, n, x.stride(0), _stream())), "idiff_softmax_rows")
    return x


# ------------------------------------------------------------------------------------------------
# CLIP text encoder pieces (csrc/clip.cu)
# ------------------------------------------------------------------------------------------------
def embed_tokens(ids: torch.Tensor, tok_table: torch.Tensor, pos_table: torch.Tensor) -> torch.Tensor:
    """ids int64 (B, T); tok_table 16-bit [V, C]; pos_table 16-bit [>= T, C] -> 16-bit [B*T, C] = tok[ids] + pos[t]."""
    lib = _lib.load()
    _req(ids, torch.int64, "ids")
    _req(tok_table, HALF, "tok_table")
    _req(pos_table, HALF, "pos_table")
    B, T = ids.shape
    V, Cc = tok_table.shape
    if pos_table.shape[0] < T or pos_table.shape[1] != Cc or not (tok_table.is_contiguous() and pos_table.is_contiguous()):
        raise _lib.IdiffError(f"embed_tokens: position table {tuple(pos_table.shape)} does not cover {T} tokens of width {Cc}")
    ids = ids.contiguous()
    out = torch.empty((B * T, Cc), dtype=HALF, device=ids.device)
    check(lib.idiff_embed_tokens(ids.data_ptr(), tok_table.data_ptr(), pos_table.data_ptr(), out.data_ptr(), B * T, T, V, Cc,
                                 _stream()), "idiff_embed_tokens")
    return out


def causal_attention_small(qkv: torch.Tensor, *, batch: int, tokens: int, heads: int, head_dim: int, scale: float,
                           key_len: Optional[torch.Tensor] = None) -> torch.Tensor:
    """qkv 16-bit [batch*tokens, 3*heads*head_dim] (q | k | v) -> 16-bit [batch*tokens, heads*head_dim]: causal
    softmax attention for short sequences (CLIP text: 77 tokens, 12 heads of 64)."""
    lib = _lib.load()
    _req(qkv, HALF, "qkv")
    C_ = heads * head_dim
    if qkv.dim() != 2 or qkv.shape[0] != batch * tokens or qkv.shape[1] < 3 * C_:
        raise _lib.IdiffError(f"causal_attention_small: qkv {tuple(qkv.shape)} vs batch {batch} tokens {tokens} width {3 * C_}")
    if key_len is not None:
        _req(key_len, torch.int32, "key_len")
        if key_len.numel() != batch:
            raise _lib.IdiffError("causal_attention_small: key_len must hold one length per sequence")
    out = torch.empty((batch * tokens, C_), dtype=HALF, device=qkv.device)
    flops = 2.0 * batch * heads * tokens * tokens * head_dim  # (causal: half of 4 N^2 d)
    check(_launch("attention_causal_small", flops, 2.0 * (qkv.numel() + out.numel()), lambda: lib.idiff_causal_attention_small(
        qkv.data_ptr(), qkv[:, C_:].data_ptr(), qkv[:, 2 * C_:].data_ptr(), out.data_ptr(), _ptr(key_len), qkv.stride(0),
        out.stride(0), batch, tokens, heads, head_dim, float(scale), _stream())), "idiff_causal_attention_small")
    return out


# ------------------------------------------------------------------------------------------------
# instance-isolation attention mask (utils/input.py:34-37, attention.py:203-247)
# ------------------------------------------------------------------------------------------------
def boxes_to_attmask(boxes: torch.Tensor, counts: torch.Tensor, size: int = 64) -> torch.Tensor:
    """boxes fp32 (B, max_objs, 4) xyxy in [0, 1], counts int32 (B,) instances per sample -> att_masks fp32
    (B, max_objs, size, size) exactly as utils/input.py:34-37 rasterises them on the host."""
    lib = _lib.load()
    _req(boxes, torch.float32, "boxes")
    _req(counts, torch.int32, "counts")
    B, K, _ = boxes.shape
    boxes = boxes.contiguous()
    att = torch.empty((B, K, size, size), dtype=torch.float32, device=boxes.device)
    check(lib.idiff_boxes_to_attmask(boxes.data_ptr(), counts.data_ptr(), att.data_ptr(), B, K, size, _stream()),
          "idiff_boxes_to_attmask")
    return att


def attmask_words(att_masks: torch.Tensor, active: torch.Tensor, tail: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """att_masks fp32 (B, n_objs, S, S), active int32 (B,) -> (mask_q int32 [B, S*S], mask_k int32 [B, S*S + 4*n_objs +
    tail]) for ops.attention(mask=...)."""
    lib = _lib.load()
    _req(att_masks, torch.float32, "att_masks")
    _req(active, torch.int32, "active")
    B, K, S, S2 = att_masks.shape
    att_masks = att_masks.contiguous()
    P = S * S2
    mq = torch.empty((B, P), dtype=torch.int32, device=att_masks.device)
    mk = torch.empty((B, P + 4 * K + tail), dtype=torch.int32, device=att_masks.device)
    check(lib.idiff_attmask_words(att_masks.data_ptr(), active.data_ptr(), mq.data_ptr(), mk.data_ptr(), B, K, P, tail,
                                  _stream()), "idiff_attmask_words")
    return mq, mk
