"""SD1.5 UNet with UniFusion fusers and ScaleU -- drop-in for the reference's
ldm/modules/diffusionmodules/openaimodel.py (same class names, constructor kwargs, forward
signatures, attributes and the 1199 state_dict keys of SURVEY.md appendix B), executing on
libidiff_b200.so.

GPU-first restructuring of `UNetModel.forward_single_input` (openaimodel.py:482-563); each item is
exact in real arithmetic (SURVEY.md section 7):
  * activations stay fp16 NHWC == token-major from the first conv to the last; every conv / linear
    is one wgmma GEMM whose epilogue carries bias, time-embedding add, residual, gate, GEGLU;
  * step-invariant work is hoisted and cached: UniFusion object tokens and their per-fuser K/V,
    the text K/V of the 16 cross-attentions (one batched GEMM), and per step one batched GEMM for
    the 22 ResBlock time-embedding projections;
  * fusers are skipped entirely on alpha=0 steps (scale == 0 => exact identity);
  * cond / uncond (and MIS trajectories) run as ONE batched forward (`forward_batched`), optionally
    replayed from a CUDA graph.
"""
from __future__ import annotations

import os
from copy import deepcopy
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .... import ops
from ....packing import pack_conv1x1, pack_conv3x3, pack_conv3x3_taps
from ...util import instantiate_from_config
from .._base import half, PackedModule, f32, nchw_to_nhwc16, nhwc16_to_nchw, w16
from ..attention import SpatialTransformer, attention_mask_words
from .util import zero_module


def conv_nd(dims, *args, **kwargs):
    if dims != 2:
        raise ValueError(f"unsupported dimensions: {dims}")
    return nn.Conv2d(*args, **kwargs)


def linear(*args, **kwargs):
    return nn.Linear(*args, **kwargs)


def normalization(channels):
    """GroupNorm32 (util.py:208-225): 32 groups, eps 1e-5, fp32 statistics."""
    return nn.GroupNorm(32, channels)


def Fourier_filter(x_in, threshold, scale):
    """openaimodel.py:25-48 for threshold == 1 (the only value the model uses), evaluated in
    closed form by idiff_scaleu_concat: x + (scale-1) * P_low(x)."""
    if threshold != 1:
        raise NotImplementedError("Fourier_filter: only threshold=1 is on the InstanceDiffusion path")
    x16, B, H, W = nchw_to_nhwc16(x_in)
    C = x16.shape[-1]
    dummy_h = torch.zeros((B * H * W, 8), dtype=half(), device=x16.device)
    ones = torch.ones(8, dtype=torch.float32, device=x16.device)
    out = ops.scaleu_concat(dummy_h, x16, ones, float(scale), batch=B, height=H, width=W)
    return nhwc16_to_nchw(out[:, 8:], B, H, W, x_in.dtype)


class TimestepBlock(PackedModule):
    """Any module whose forward takes the timestep embedding as second argument."""


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """openaimodel.py:62-79 (module-level API; the UNet fast path walks the children itself)."""

    def forward(self, x, emb, context, objs, grounding_input=None, drop_box_mask=False):
        for layer in self:
            if isinstance(layer, TimestepBlock):
                x = layer(x, emb)
            elif isinstance(layer, SpatialTransformer):
                x = layer(x, context, objs, grounding_input, drop_box_mask=drop_box_mask)
            elif isinstance(layer, nn.Conv2d):
                x = _conv3x3_module_forward(layer, x)
            else:
                x = layer(x)
        return x


def _conv3x3_module_forward(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """nn.Conv2d(4, 320, 3, padding=1) holder of input_blocks[0] run through the conv kernel."""
    x16, B, H, W = nchw_to_nhwc16(x)
    cin = x16.shape[-1]
    cpad = (cin + 63) // 64 * 64
    if cpad != cin:
        xp = torch.zeros((x16.shape[0], cpad), dtype=half(), device=x16.device)
        xp[:, :cin] = x16
        x16 = xp
    wp = _pack_conv3x3_padded(conv.weight, cpad)
    y = ops.gemm(x16, wp, f32(conv.bias), conv=(B, H, W, cpad))
    return nhwc16_to_nchw(y, B, H, W, x.dtype)


def _pack_conv3x3_padded(weight: torch.Tensor, cin_pad: int) -> torch.Tensor:
    cout, cin = weight.shape[:2]
    w = torch.zeros((cout, cin_pad, 3, 3), dtype=half(), device=weight.device)
    w[:, :cin] = weight.detach().to(half())
    return pack_conv3x3(w)


class Upsample(PackedModule):
    """openaimodel.py:82-110: nearest 2x then conv3x3."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if use_conv:
            self.conv = conv_nd(dims, self.channels, self.out_channels, 3, padding=padding)

    def _pack(self):
        if not self.use_conv:
            return {}
        return {"w": pack_conv3x3(w16(self.conv.weight)), "b": f32(self.conv.bias)}

    def _fwd(self, x16, B, H, W):
        up = ops.upsample_nearest2x(x16, B, H, W)
        if not self.use_conv:
            return up
        p = self.pk()
        return ops.gemm(up, p["w"], p["b"], conv=(B, 2 * H, 2 * W, self.channels))

    def forward(self, x):
        assert x.shape[1] == self.channels
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, 2 * H, 2 * W, x.dtype)


class Downsample(PackedModule):
    """openaimodel.py:113-141: conv3x3 stride 2 padding 1."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if not use_conv:
            raise NotImplementedError("Downsample(use_conv=False) is not on the InstanceDiffusion path")
        self.op = conv_nd(dims, self.channels, self.out_channels, 3, stride=2, padding=padding)

    def _pack(self):
        return {"w": pack_conv3x3(w16(self.op.weight)), "b": f32(self.op.bias)}

    def _fwd(self, x16, B, H, W):
        p = self.pk()
        cols = ops.im2col_s2(x16, B, H, W)
        return ops.gemm(cols, p["w"], p["b"])

    def forward(self, x):
        assert x.shape[1] == self.channels
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, H // 2, W // 2, x.dtype)


class ResBlock(TimestepBlock):
    """openaimodel.py:144-257 (no up/down, no scale-shift norm -- the SD1.5 configuration):
    GN+SiLU -> conv3x3 (+bias +emb in the epilogue) -> GN+SiLU -> conv3x3 (+bias +skip in the
    epilogue); skip = identity or a 1x1 conv GEMM."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False,
                 use_scale_shift_norm=False, dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        if up or down or use_scale_shift_norm or use_conv:
            raise NotImplementedError("ResBlock up/down/scale_shift/use_conv are not on the InstanceDiffusion path")
        self.channels = channels
        self.emb_channels = emb_channels
        self.dropout = dropout
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.use_checkpoint = use_checkpoint
        self.use_scale_shift_norm = use_scale_shift_norm
        self.updown = False
        self.in_layers = nn.Sequential(normalization(channels), nn.SiLU(),
                                       conv_nd(dims, channels, self.out_channels, 3, padding=1))
        self.h_upd = self.x_upd = nn.Identity()
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(conv_nd(dims, self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = conv_nd(dims, channels, self.out_channels, 1)

    def _pack(self):
        p = {
            "g1": f32(self.in_layers[0].weight), "b1": f32(self.in_layers[0].bias),
            "w1": pack_conv3x3(w16(self.in_layers[2].weight)), "cb1": f32(self.in_layers[2].bias),
            "we": w16(self.emb_layers[1].weight), "be": f32(self.emb_layers[1].bias),
            "g2": f32(self.out_layers[0].weight), "b2": f32(self.out_layers[0].bias),
            "w2": pack_conv3x3(w16(self.out_layers[3].weight)), "cb2": f32(self.out_layers[3].bias),
        }
        if not isinstance(self.skip_connection, nn.Identity):
            p["ws"] = pack_conv1x1(w16(self.skip_connection.weight))
            p["bs"] = f32(self.skip_connection.bias)
        return p

    def _fwd(self, x16, B, H, W, emb_out):
        """x16 fp16 [B*H*W, Cin]; emb_out fp16 [B, Cout] view = Linear(SiLU(emb)) (openaimodel.py:246)."""
        p = self.pk()
        hw = H * W
        h = ops.groupnorm(x16, p["g1"], p["b1"], batch=B, hw=hw, groups=32, eps=1e-5, silu=True)
        h = ops.gemm(h, p["w1"], p["cb1"], conv=(B, H, W, self.channels), rowadd=emb_out)
        h = ops.groupnorm(h, p["g2"], p["b2"], batch=B, hw=hw, groups=32, eps=1e-5, silu=True)
        skip = x16 if "ws" not in p else ops.gemm(x16, p["ws"], p["bs"])
        return ops.gemm(h, p["w2"], p["cb2"], conv=(B, H, W, self.out_channels), residual=skip)

    def forward(self, x, emb):
        return self._forward(x, emb)

    def _forward(self, x, emb):
        x16, B, H, W = nchw_to_nhwc16(x)
        p = self.pk()
        e16 = ops.silu(emb.to(half()).contiguous())
        emb_out = ops.gemm(e16, p["we"], p["be"])
        return nhwc16_to_nchw(self._fwd(x16, B, H, W, emb_out), B, H, W, x.dtype)


class UNetModel(PackedModule):
    # bounds of the hoisted-tensor caches: text K/V and object K/V entries (one per distinct input), concatenations
    # (one per combination of inputs in a batched forward); a cache that reaches its bound is cleared
    hoist_cache_entries = 64
    cat_cache_entries = 6
    # memory pool token (torch.cuda.graph_pool_handle()) that new graph captures share; None: a private pool each
    graph_pool = None

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks,
                 attention_resolutions, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2,
                 use_checkpoint=False, num_heads=8, use_scale_shift_norm=False, transformer_depth=1,
                 context_dim=None, fuser_type=None, inpaint_mode=False, grounding_downsampler=None,
                 grounding_tokenizer=None, sd_v1_5=False, efficient_attention=False):
        super().__init__()
        self.image_size = image_size
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = attention_resolutions
        self.dropout = dropout
        self.channel_mult = channel_mult
        self.conv_resample = conv_resample
        self.use_checkpoint = use_checkpoint
        self.num_heads = num_heads
        self.context_dim = context_dim
        self.fuser_type = fuser_type
        self.inpaint_mode = inpaint_mode
        self.sd_v1_5 = sd_v1_5
        assert fuser_type in ["gatedSA", "gatedSA2", "gatedCA"]
        if fuser_type != "gatedSA":
            raise NotImplementedError("only fuser_type='gatedSA' exists in the reference's attention.py")
        self.efficient_attention = efficient_attention
        self.grounding_tokenizer_input = None  # set externally (inference.py:307)
        self.enable_freeu = False
        self.enable_scaleu = True
        self.enable_se_scaleu = False

        time_embed_dim = model_channels * 4
        self.time_embed = nn.Sequential(linear(model_channels, time_embed_dim), nn.SiLU(),
                                        linear(time_embed_dim, time_embed_dim))
        self.downsample_net = None
        self.additional_channel_from_downsampler = 0
        self.first_conv_restorable = True

        self.input_blocks = nn.ModuleList(
            [TimestepEmbedSequential(conv_nd(dims, in_channels, model_channels, 3, padding=1))])
        input_block_chans = [model_channels]
        ch = model_channels
        ds = 1

        def make_st(ch_):
            return SpatialTransformer(ch_, key_dim=context_dim, value_dim=context_dim, n_heads=num_heads,
                                      d_head=ch_ // num_heads, depth=transformer_depth, fuser_type=fuser_type,
                                      use_checkpoint=use_checkpoint, efficient_attention=efficient_attention)

        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [ResBlock(ch, time_embed_dim, dropout, out_channels=mult * model_channels, dims=dims,
                                   use_checkpoint=use_checkpoint, use_scale_shift_norm=use_scale_shift_norm)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    layers.append(make_st(ch))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                input_block_chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, conv_resample, dims=dims, out_channels=ch)))
                input_block_chans.append(ch)
                ds *= 2

        self.middle_block = TimestepEmbedSequential(
            ResBlock(ch, time_embed_dim, dropout, dims=dims, use_checkpoint=use_checkpoint,
                     use_scale_shift_norm=use_scale_shift_norm),
            make_st(ch),
            ResBlock(ch, time_embed_dim, dropout, dims=dims, use_checkpoint=use_checkpoint,
                     use_scale_shift_norm=use_scale_shift_norm))

        self.output_blocks = nn.ModuleList([])
        idx = 0
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = input_block_chans.pop()
                layers = [ResBlock(ch + ich, time_embed_dim, dropout, out_channels=model_channels * mult, dims=dims,
                                   use_checkpoint=use_checkpoint, use_scale_shift_norm=use_scale_shift_norm)]
                self.register_parameter('scaleu_b_{}'.format(idx), nn.Parameter(torch.zeros(ch)))
                self.register_parameter('scaleu_s_{}'.format(idx), nn.Parameter(torch.zeros(1)))
                idx += 1
                ch = model_channels * mult
                if ds in attention_resolutions:
                    layers.append(make_st(ch))
                if level and i == num_res_blocks:
                    layers.append(Upsample(ch, conv_resample, dims=dims, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))

        self.out = nn.Sequential(normalization(ch), nn.SiLU(),
                                 zero_module(conv_nd(dims, model_channels, out_channels, 3, padding=1)))
        self.position_net = instantiate_from_config(grounding_tokenizer)

        # hoisted, step-invariant tensors (keyed caches)
        self._ctx_cache: Dict = {}
        self._obj_cache: Dict = {}
        self._cat_cache: Dict = {}
        self._graphs: Dict = {}
        self._in_packs: Dict = {}
        self.use_cuda_graph = os.environ.get("IDIFF_CUDA_GRAPH", "1") != "0"

    # ------------------------------------------------------------------------------------------
    # reference side effects
    # ------------------------------------------------------------------------------------------
    def restore_first_conv_from_SD(self):
        """openaimodel.py:469-480: on the first alpha == 0 step the input conv is permanently replaced
        by the SD1.5 weights shipped in pretrained/.  The reference re-reads the file on every such
        step; the result is the same tensor each time, so it is loaded once."""
        if not self.first_conv_restorable:
            return
        if getattr(self, "_first_conv_restored", False):
            return
        self.set_sd_first_conv(self.load_sd_first_conv())

    def load_sd_first_conv(self) -> Dict[str, torch.Tensor]:
        """The SD1.5 input-conv state dict restore_first_conv_from_SD swaps in, read from pretrained/ (cwd-relative
        as in the reference, openaimodel.py:476) or $IDIFF_PRETRAINED_DIR.  Swaps nothing."""
        name = "SD_v1_5_input_conv_weight_bias.pth" if self.sd_v1_5 else "SD_input_conv_weight_bias.pth"
        path = os.path.join("pretrained", name)
        if not os.path.exists(path):
            alt = os.environ.get("IDIFF_PRETRAINED_DIR")
            if alt and os.path.exists(os.path.join(alt, name)):
                path = os.path.join(alt, name)
            else:
                raise FileNotFoundError(
                    f"{path} not found (cwd-relative as in the reference, openaimodel.py:476); "
                    "set IDIFF_PRETRAINED_DIR or call set_sd_first_conv(state_dict)")
        return torch.load(path, map_location="cpu")

    def set_sd_first_conv(self, sd_weights: Dict[str, torch.Tensor]):
        conv = self.input_blocks[0][0]
        device = conv.weight.device
        self.first_conv_state_dict = deepcopy(conv.state_dict())
        new = conv_nd(2, 4, 320, 3, padding=1)
        new.load_state_dict(sd_weights)
        self.input_blocks[0][0] = new.to(device)
        self._first_conv_restored = True
        # The packed first-conv weights of both states are kept alive side by side (the captured CUDA
        # graphs of either state point at them), so swapping costs nothing and invalidates nothing --
        # unless different SD weights than last time are supplied.
        if getattr(self, "_sd_conv_src", None) is not sd_weights:
            self._sd_conv_src = sd_weights
            self._in_packs.pop((True, False), None)
            self._in_packs.pop((True, True), None)
            for k in [k for k in self._graphs if k[-1]]:
                del self._graphs[k]

    def undo_first_conv_restore(self):
        """Not in the reference (whose swap is permanent within a process): lets a long-lived server /
        the benchmark run several `sample()` calls on one model object."""
        if getattr(self, "_first_conv_restored", False):
            conv = conv_nd(2, 4, 320, 3, padding=1)  # a new module: packs built from the SD conv keep their tensors
            conv.load_state_dict(self.first_conv_state_dict)
            self.input_blocks[0][0] = conv.to(self.input_blocks[0][0].weight.device)
            self._first_conv_restored = False

    def _in_conv_pack(self, restored: Optional[bool] = None, taps: bool = False):
        """Packed input conv of the model's current first-conv state, or (restored=True / False) of the SD1.5 /
        the model's own conv whatever the current state is.  The SD weights are the ones last given to
        set_sd_first_conv, else load_sd_first_conv().  taps: in the layout of ops.conv_in_select instead of the
        conv GEMM's."""
        cur = bool(getattr(self, "_first_conv_restored", False))
        key = cur if restored is None else bool(restored)
        hit = self._in_packs.get((key, taps))
        if hit is None:
            conv0 = self.input_blocks[0][0]
            if key == cur:
                w, b = conv0.weight, conv0.bias
            else:
                sd = self.first_conv_state_dict if cur else getattr(self, "_sd_conv_src", None)
                if sd is None:
                    sd = self.load_sd_first_conv()
                w, b = sd["weight"].to(conv0.weight.device), sd["bias"].to(conv0.weight.device)
            with torch.no_grad():
                hit = (pack_conv3x3_taps(w.detach().to(half())) if taps else _pack_conv3x3_padded(w, 64), f32(b))
            self._in_packs[(key, taps)] = hit
        return hit

    def _in_conv_taps(self):
        """((w0, b0, w1, b1) of ops.conv_in_select: the model's own input conv and the SD1.5 one, whether the SD1.5
        weights exist).  Without them both sets are the model's own conv, and no image may select the second."""
        own = self._in_conv_pack(False, taps=True)
        try:
            return own + self._in_conv_pack(True, taps=True), True
        except FileNotFoundError:
            return own + own, False

    def _drop_derived(self):
        """Everything computed from the weights: packed first conv, captured graphs, hoisted text K/V and
        object tokens / per-fuser K/V (including the null-branch entry)."""
        if hasattr(self, "_in_packs"):
            self._in_packs.clear()
            self._graphs.clear()
            self._ctx_cache.clear()
            self._obj_cache.clear()
            self._cat_cache.clear()

    def _apply(self, fn, *a, **k):
        self._drop_derived()
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._drop_derived()
        return super()._load_from_state_dict(*a, **k)

    def invalidate_pack(self):
        self._drop_derived()
        return super().invalidate_pack()

    # ------------------------------------------------------------------------------------------
    # packing
    # ------------------------------------------------------------------------------------------
    def _resblocks(self) -> List[ResBlock]:
        return [m for m in self.modules() if isinstance(m, ResBlock)]

    def _transformers(self) -> List[SpatialTransformer]:
        return [m for m in self.modules() if isinstance(m, SpatialTransformer)]

    def _pack(self):
        p = {
            "wt0": w16(self.time_embed[0].weight), "bt0": f32(self.time_embed[0].bias),
            "wt2": w16(self.time_embed[2].weight), "bt2": f32(self.time_embed[2].bias),
            "g_out": f32(self.out[0].weight), "b_out": f32(self.out[0].bias),
            "w_out": pack_conv3x3(w16(self.out[2].weight)), "cb_out": f32(self.out[2].bias),
        }
        # all 22 ResBlock emb projections as one GEMM (openaimodel.py:199-205,246)
        rbs = self._resblocks()
        p["w_emb_all"] = torch.cat([w16(rb.emb_layers[1].weight) for rb in rbs], 0).contiguous()
        p["b_emb_all"] = torch.cat([f32(rb.emb_layers[1].bias) for rb in rbs], 0).contiguous()
        offs, o = {}, 0
        for rb in rbs:
            offs[id(rb)] = (o, o + rb.out_channels)
            o += rb.out_channels
        p["emb_offs"] = offs
        # all 16 cross-attention K/V projections of the text context as one GEMM (attention.py:122-123)
        blocks = [blk for st in self._transformers() for blk in st.transformer_blocks]
        p["w_ctx_all"] = torch.cat([blk.attn2.pk()["wkv"] for blk in blocks], 0).contiguous()
        coffs, o = {}, 0
        for blk in blocks:
            n = blk.attn2.pk()["wkv"].shape[0]
            coffs[id(blk)] = (o, o + n)
            o += n
        p["ctx_offs"] = coffs
        # ScaleU factors (openaimodel.py:524-525): tanh(b)+1 per channel, tanh(s)+1 scalar
        p["scaleu_b"] = [(torch.tanh(getattr(self, f"scaleu_b_{i}").detach().float()) + 1).contiguous()
                         for i in range(len(self.output_blocks))]
        p["ones"] = torch.ones(max(getattr(self, f"scaleu_b_{i}").numel() for i in range(len(self.output_blocks))),
                               dtype=torch.float32, device=p["g_out"].device)
        p["scaleu_s"] = [float(torch.tanh(getattr(self, f"scaleu_s_{i}").detach().float().cpu()) + 1)
                         for i in range(len(self.output_blocks))]
        return p

    # ------------------------------------------------------------------------------------------
    # hoisted step-invariant tensors
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _tkey(t: torch.Tensor):
        return (t.data_ptr(), t._version, tuple(t.shape), t.dtype)

    def context_kv(self, context: torch.Tensor) -> torch.Tensor:
        """K|V of all 16 cross-attentions for a (B,77,768) context: [B*77, sum 2C], cached."""
        key = self._tkey(context)
        hit = self._ctx_cache.get(key)
        if hit is not None:
            return hit[1]
        p = self.pk()
        c16 = context.reshape(-1, context.shape[-1]).to(half()).contiguous()
        kv = ops.gemm(c16, p["w_ctx_all"])
        if len(self._ctx_cache) > self.hoist_cache_entries:
            self._ctx_cache.clear()
            self._cat_cache.clear()
        self._ctx_cache[key] = (context, kv)  # keep `context` alive so the key stays unique
        return kv

    def object_kv(self, grounding_input: Optional[dict]):
        """UniFusion tokens -> (per-fuser K|V ([Bo*184, 2C] each), Bo, n_obj, mask words or None), cached per
        grounding_input dict.  `None` selects the null (CFG-uncond) tokens, which are a pure function of the
        weights.  Mask words: the instance-isolation mask of the 64x64-level fusers (attention.py:187-255) when the
        grounding input carries `att_masks` and the model was built without `efficient_attention`."""
        if grounding_input is None:
            gti = self.grounding_tokenizer_input
            gi = gti.get_null_input()
            # the null tokens depend on the weights and on the shapes prepare() remembered
            key = ("null", gti.batch, gti.max_box, gti.in_dim, gti.dim_scribbles, gti.dim_polygons,
                   str(gi["boxes"].device))
        else:
            gi = grounding_input
            key = self._obj_key(gi)
        hit = self._obj_cache.get(key)
        if hit is not None:
            return hit[1]
        objs16, Bo, n_obj, drop_box_mask = self.position_net._tokens(gi["boxes"], gi["masks"], gi["positive_embeddings"],
                                                                    gi["scribbles"], gi["polygons"], gi["segs"], gi["points"])
        blocks = [blk for st in self._transformers() for blk in st.transformer_blocks]
        kvs = [blk.fuser.project_objs(objs16) for blk in blocks]
        mask = attention_mask_words(blocks[0].fuser, gi, drop_box_mask, Bo, 64 * 64, n_obj)
        if len(self._obj_cache) > self.hoist_cache_entries:
            self._obj_cache.clear()
            self._cat_cache.clear()
        val = (kvs, Bo, n_obj, mask)
        self._obj_cache[key] = (gi, val)
        return val

    def _obj_key(self, gi: dict):
        return tuple(self._tkey(gi[k]) for k in ("boxes", "masks", "positive_embeddings", "scribbles", "polygons",
                                                "segs", "points", "att_masks") if gi.get(k) is not None)

    def drop_hoisted(self, inputs: List[dict], keep: List[dict] = ()):
        """Drop the hoisted tensors of `inputs` (text K/V of their context, object K/V of their grounding input) and
        every batch concatenation that holds one of them, except those that the inputs in `keep` share.  What a
        server calls when a request finishes."""
        def keys(ins):
            return ({self._tkey(i["context"]) for i in ins},
                    {self._obj_key(i["grounding_input"]) for i in ins if i.get("grounding_input") is not None})
        ctx_keys, obj_keys = keys(inputs)
        kept_ctx, kept_obj = keys(keep)
        gone = [self._ctx_cache.pop(k) for k in ctx_keys - kept_ctx if k in self._ctx_cache]
        gone_obj = [self._obj_cache.pop(k) for k in obj_keys - kept_obj if k in self._obj_cache]
        ids = {id(v[1]) for v in gone} | {id(v[1][0]) for v in gone_obj} | {id(v[1][3]) for v in gone_obj if v[1][3] is not None}
        for k in [k for k in self._cat_cache if ids & set(k[2] + k[3] + k[4])]:
            del self._cat_cache[k]

    def trim_concats(self, keep: int):
        """Keep only the `keep` most recently used batch concatenations of the hoisted tensors."""
        for k in list(self._cat_cache)[:max(len(self._cat_cache) - int(keep), 0)]:
            del self._cat_cache[k]

    def clear_hoisted(self):
        """Drop the per-sample hoisted tensors (text K/V, UniFusion tokens / object K/V, their concatenations);
        captured graphs stay.  What a server calls between requests."""
        self._ctx_cache.clear()
        self._obj_cache.clear()
        self._cat_cache.clear()

    def trim_hoisted(self):
        """Drop the batch concatenations of the hoisted tensors, and the per-input caches where they hold more
        entries than their bound (a run with raised bounds leaves them so)."""
        self._cat_cache.clear()
        if len(self._ctx_cache) > self.hoist_cache_entries:
            self._ctx_cache.clear()
        if len(self._obj_cache) > self.hoist_cache_entries:
            self._obj_cache.clear()

    def clear_caches(self):
        self.clear_hoisted()
        self._graphs.clear()

    # ------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------
    def _fusers_active(self) -> bool:
        return any(blk.fuser.scale != 0 for st in self._transformers() for blk in st.transformer_blocks)

    def _core(self, x: torch.Tensor, t: torch.Tensor, ctx_kv_all: torch.Tensor, M: int,
              obj_kvs: Optional[List[torch.Tensor]], n_obj: int, mask=None, fuser_scale=None,
              n_restored=None) -> torch.Tensor:
        """x fp32 (B,4,H,W), t fp32 (B,), ctx_kv_all fp16 [B*M, sumKV], obj_kvs per-fuser [B*n_obj, 2C]
        (or None on alpha=0 steps) -> eps fp32 (B,4,H,W).  fuser_scale: None (each fuser's `.scale`), a float or
        an fp32 [B] tensor of per-image scales.  n_restored: None (the model's first-conv state for every image),
        the number of trailing images that take the SD1.5 input conv, the others the model's own, or an int32 [B]
        device tensor of per-image flags (1: the SD1.5 conv) for ops.conv_in_select."""
        p = self.pk()
        B, _, H, W = x.shape
        # time embedding (openaimodel.py:497-498) ; SiLU of emb_layers[0] folded into the last epilogue
        te = ops.timestep_embedding(t, self.model_channels)
        e = ops.gemm(te, p["wt0"], p["bt0"], silu=True)
        e = ops.gemm(e, p["wt2"], p["bt2"], silu=True)
        emb_all = ops.gemm(e, p["w_emb_all"], p["b_emb_all"])

        def emb_of(rb):
            a, b = p["emb_offs"][id(rb)]
            return emb_all[:, a:b]

        blk_idx = [0]

        def run_st(st: SpatialTransformer, h, hh, ww):
            ctx_kvs, okvs = [], []
            for blk in st.transformer_blocks:
                a, b = p["ctx_offs"][id(blk)]
                ctx_kvs.append(ctx_kv_all[:, a:b])
                okvs.append(obj_kvs[blk_idx[0]] if obj_kvs is not None else None)
                blk_idx[0] += 1
            return st._fwd(h, B, hh, ww, ctx_kvs, M, okvs if obj_kvs is not None else None, n_obj, B, mask=mask,
                           fuser_scale=fuser_scale)

        def run_block(seq, h, hh, ww):
            for layer in seq:
                if isinstance(layer, ResBlock):
                    h = layer._fwd(h, B, hh, ww, emb_of(layer))
                elif isinstance(layer, SpatialTransformer):
                    h = run_st(layer, h, hh, ww)
                elif isinstance(layer, Downsample):
                    h = layer._fwd(h, B, hh, ww)
                    hh, ww = hh // 2, ww // 2
                elif isinstance(layer, Upsample):
                    h = layer._fwd(h, B, hh, ww)
                    hh, ww = hh * 2, ww * 2
                else:
                    raise TypeError(f"unexpected layer {type(layer)}")
            return h, hh, ww

        if isinstance(n_restored, torch.Tensor):
            h = ops.conv_in_select(x, *self._in_conv_taps()[0], n_restored)
        elif n_restored is None or n_restored in (0, B):
            x16 = ops.nchw_f32_to_nhwc_f16(x, 64)
            w_in, b_in = self._in_conv_pack(None if n_restored is None else n_restored == B)
            h = ops.gemm(x16, w_in, b_in, conv=(B, H, W, 64))
        else:  # one conv GEMM per first-conv state, each on its contiguous range of images
            x16 = ops.nchw_f32_to_nhwc_f16(x, 64)
            h = torch.empty((B * H * W, self.model_channels), dtype=half(), device=x.device)
            for b0, nb, restored in ((0, B - n_restored, False), (B - n_restored, n_restored, True)):
                w_in, b_in = self._in_conv_pack(restored)
                rows = slice(b0 * H * W, (b0 + nb) * H * W)
                ops.gemm(x16[rows], w_in, b_in, conv=(nb, H, W, 64), out=h[rows])
        hh, ww = H, W
        hs = [(h, hh, ww)]
        for module in list(self.input_blocks)[1:]:
            h, hh, ww = run_block(module, h, hh, ww)
            hs.append((h, hh, ww))
        h, hh, ww = run_block(self.middle_block, h, hh, ww)
        for idx, module in enumerate(self.output_blocks):
            skip, sh, sw = hs.pop()
            assert (sh, sw) == (hh, ww)
            if self.enable_freeu or self.enable_se_scaleu:
                raise NotImplementedError("FreeU / SE-ScaleU skip rescaling (openaimodel.py:519-560) is not on "
                                          "the shipped sampling path; only enable_scaleu is implemented")
            if self.enable_scaleu:
                b1, s_ = p["scaleu_b"][idx], p["scaleu_s"][idx]
            else:  # plain torch.cat([h, hs.pop()], dim=1): unit factors make the pass an exact copy
                b1, s_ = p["ones"][: h.shape[-1]], 1.0
            h = ops.scaleu_concat(h, skip, b1, s_, batch=B, height=hh, width=ww)
            h, hh, ww = run_block(module, h, hh, ww)
        h = ops.groupnorm(h, p["g_out"], p["b_out"], batch=B, hw=hh * ww, groups=32, eps=1e-5, silu=True)
        eps = torch.empty((B, self.out_channels, hh, ww), dtype=torch.float32, device=x.device)
        ops.gemm(h, p["w_out"], p["cb_out"], conv=(B, hh, ww, self.model_channels), out_nchw=eps)
        return eps

    def _gather_inputs(self, inputs: List[dict], active: Optional[bool] = None):
        """Concatenate independent forwards (cond / uncond / MIS trajectories) along the batch.  The step-invariant
        parts -- text K/V, per-fuser object K/V, mask words -- are concatenated once per combination of inputs and
        reused on every later step (the same tensor objects come back, which lets `_CoreGraph.replay` skip its copies
        as well): 17-19 torch.cat launches and as many copies per forward otherwise.  active: whether the fusers run
        (default: any fuser has a non-zero `.scale`)."""
        xs, ts, ctxs, okv_lists, masks, bs = [], [], [], [], [], []
        if active is None:
            active = self._fusers_active()
        n_obj = 0
        for inp in inputs:
            x = inp["x"]
            b = x.shape[0]
            bs.append(b)
            xs.append(x.float())
            ts.append(inp["timesteps"].float().reshape(-1).expand(b) if inp["timesteps"].numel() == 1
                      else inp["timesteps"].float())
            ctxs.append(self.context_kv(inp["context"]))
            if active:
                kvs, Bo, n_obj_i, mask_i = self.object_kv(inp.get("grounding_input"))
                masks.append((mask_i, b))
                if n_obj and n_obj_i != n_obj:
                    raise ValueError(f"inputs of one batched forward carry different object-token counts "
                                     f"({n_obj} vs {n_obj_i}); prepare() them with the same max_box")
                n_obj = n_obj_i
                if Bo != b and Bo != 1:
                    raise ValueError(f"grounding batch {Bo} does not match latent batch {b}")
                okv_lists.append((kvs, Bo))
        M = inputs[0]["context"].shape[1]
        x = xs[0].contiguous() if len(inputs) == 1 else torch.cat(xs, 0)
        t = ts[0].contiguous() if len(inputs) == 1 else torch.cat(ts, 0)
        # the hoisted tensors above are cached objects: their identities (and the batch sizes) name the combination
        key = (active, tuple(bs), tuple(id(c) for c in ctxs), tuple(id(k) for k, _ in okv_lists),
               tuple(id(m) for m, _ in masks))
        hit = self._cat_cache.pop(key, None)
        if hit is not None:
            self._cat_cache[key] = hit  # most recently used last (trim_concats)
            _, ctx, okv, mask = hit
            return x, t, ctx, M, okv, n_obj, mask
        ctx = ctxs[0] if len(inputs) == 1 else torch.cat(ctxs, 0)
        okv = None
        if active:
            per_input = []
            for (kvs, Bo), b in zip(okv_lists, bs):
                if Bo != b:
                    kvs = [kv.view(1, n_obj, -1).expand(b, n_obj, kv.shape[-1]).reshape(b * n_obj, -1) for kv in kvs]
                per_input.append(kvs)
            okv = per_input[0] if len(inputs) == 1 else \
                [torch.cat([l[i] for l in per_input], 0) for i in range(len(per_input[0]))]
        # instance-isolation mask words: inputs without a mask (the CFG null branch) get all-ones words
        mask = None
        if any(m is not None for m, _ in masks):
            dev = xs[0].device
            mqs, mks = [], []
            for m, b in masks:
                if m is None:
                    mqs.append(torch.full((b, 64 * 64), -1, dtype=torch.int32, device=dev))
                    mks.append(torch.full((b, 64 * 64 + n_obj), -1, dtype=torch.int32, device=dev))
                else:
                    mq, mk = m
                    mqs.append(mq if mq.shape[0] == b else mq.expand(b, -1))
                    mks.append(mk if mk.shape[0] == b else mk.expand(b, -1))
            mask = (torch.cat(mqs, 0).contiguous(), torch.cat(mks, 0).contiguous())
        if len(self._cat_cache) >= self.cat_cache_entries:  # (an entry holds the concatenated text K/V: tens of MB to ~1 GB at MIS batch sizes)
            self._cat_cache.clear()
        keep = (ctxs, [k for k, _ in okv_lists], [m for m, _ in masks])  # keeps the keyed objects (and their ids) alive
        self._cat_cache[key] = (keep, ctx, okv, mask)
        return x, t, ctx, M, okv, n_obj, mask

    @torch.no_grad()
    def forward_batched(self, inputs: List[dict], *, scales: Optional[List[float]] = None,
                        restored: Optional[List[bool]] = None, per_image_conv: bool = False) -> List[torch.Tensor]:
        """Run several independent forwards as one batch; returns one eps tensor per input.

        scales: one fuser scale per input -- what set_alpha_scale would set for a forward of that input alone --
        instead of the fusers' own `.scale`.  Equal scales run the scalar-gate path (all 0: the fusers are skipped);
        mixed scales run the fusers on every image with the gates tanh(alpha) * scale of each image.
        restored: per input, True = the SD1.5 input conv that restore_first_conv_from_SD swaps in, False = the
        model's own; the model's conv is not swapped.  Default: the model's current first-conv state.
        per_image_conv: choose each image's input conv on the device (ops.conv_in_select) from a per-image flag that,
        like the per-image scales, is a static input of the captured graph.  The count of SD1.5-conv images then
        stays out of the graph key, and the images keep their order."""
        if getattr(self, "_storage_epoch", None) != ops.STORAGE_EPOCH:  # storage type switched: derived tensors are stale
            self._drop_derived()
            self._storage_epoch = ops.STORAGE_EPOCH
        n = len(inputs)
        for arg, name in ((scales, "scales"), (restored, "restored")):
            if arg is not None and len(arg) != n:
                raise ValueError(f"forward_batched: {len(arg)} {name} for {n} inputs")
        sizes = [inp["x"].shape[0] for inp in inputs]
        if per_image_conv:
            order = list(range(n))
            cur = bool(getattr(self, "_first_conv_restored", False))
            flags = [bool(restored[i]) if restored is not None else cur for i in range(n)]
            if any(flags):
                self._in_conv_pack(True, taps=True)  # raises when no SD1.5 conv weights exist
            rows_in = torch.tensor([int(f) for f, b in zip(flags, sizes) for _ in range(b)], dtype=torch.int32)
            n_restored = rows_in.pin_memory().to(inputs[0]["x"].device, non_blocking=True)
        elif restored is None:
            order = list(range(n))
            n_restored = sum(sizes) if getattr(self, "_first_conv_restored", False) else 0
        else:  # images of the SD1.5 conv last: each input conv is one GEMM over a contiguous range of images
            order = [i for i in range(n) if not restored[i]] + [i for i in range(n) if restored[i]]
            n_restored = sum(sizes[i] for i in range(n) if restored[i])
        ins = [inputs[i] for i in order]
        fuser_scale, active = None, None
        if scales is not None:
            s = [float(scales[i]) for i in order]
            if all(v == s[0] for v in s):
                fuser_scale, active = s[0], s[0] != 0
            else:
                rows = torch.tensor([v for v, i in zip(s, order) for _ in range(sizes[i])], dtype=torch.float32)
                fuser_scale, active = rows.pin_memory().to(ins[0]["x"].device, non_blocking=True), True
        x, t, ctx, M, okv, n_obj, mask = self._gather_inputs(ins, active)
        eps = self._run_core(x, t, ctx, M, okv, n_obj, mask, fuser_scale, n_restored)
        outs = torch.split(eps, [sizes[i] for i in order], 0)
        res = [None] * n
        for j, i in enumerate(order):
            res[i] = outs[j]
        return res

    def _run_core(self, x, t, ctx, M, okv, n_obj, mask=None, fuser_scale=None, n_restored=None):
        if not self.use_cuda_graph:
            return self._core(x, t, ctx, M, okv, n_obj, mask, fuser_scale, n_restored)
        # the fuser gates scale*tanh(alpha) are kernel arguments, frozen into a captured graph: the
        # per-fuser scales (set_alpha_scale may set any value, alpha_generator's decay stage is
        # fractional) are part of the key.  Per-image scales are a static input buffer of the graph instead.
        if okv is None:
            scales = ()
        elif isinstance(fuser_scale, torch.Tensor):
            scales = ("per-image",)
        else:
            scales = tuple(float(blk.fuser.scale if fuser_scale is None else fuser_scale)
                           for st in self._transformers() for blk in st.transformer_blocks)
        if n_restored is None:
            n_restored = x.shape[0] if getattr(self, "_first_conv_restored", False) else 0
        # per-image conv flags are a static input buffer; the graph points at both packed convs (or twice at the
        # model's own while no SD1.5 weights exist)
        conv = n_restored
        if isinstance(n_restored, torch.Tensor):
            conv = "per-image" if self._in_conv_taps()[1] else "per-image, own conv only"
        # (set_sd_first_conv drops the graphs whose last key entry, the count of SD-conv images, is truthy)
        key = (tuple(x.shape), M, scales, n_obj, mask is not None, conv)
        g = self._graphs.get(key)
        if g is None:
            g = _CoreGraph(self, x, t, ctx, M, okv, n_obj, mask, fuser_scale, n_restored)
            self._graphs[key] = g
        return g.replay(x, t, ctx, okv, mask, fuser_scale, n_restored)

    def forward_single_input(self, input):
        return self.forward_batched([input])[0]

    def forward(self, input):
        return self.forward_single_input(input)


class _CoreGraph:
    """One captured CUDA graph of UNetModel._core for a fixed (batch, shapes, fuser on/off) key.
    Inputs are copied into static buffers, the graph is replayed, the static output is cloned."""

    def __init__(self, model: UNetModel, x, t, ctx, M, okv, n_obj, mask=None, fuser_scale=None, n_restored=None):
        self.x = x.clone()
        self.t = t.clone()
        self.ctx = ctx.clone()
        self.okv = [o.clone() for o in okv] if okv is not None else None
        self.mask = (mask[0].clone(), mask[1].clone()) if mask is not None else None
        # per-image fuser scales: a static input like x and t (a float or None is part of the graph key)
        self.scale = fuser_scale.clone() if isinstance(fuser_scale, torch.Tensor) else fuser_scale
        self.conv = n_restored.clone() if isinstance(n_restored, torch.Tensor) else n_restored
        model.pk()  # make sure packing (allocations + host work) happens outside capture
        for st in model._transformers():
            st.pk()
            for blk in st.transformer_blocks:
                for m in blk.modules():
                    if isinstance(m, PackedModule):
                        m.pk()
        for m in model.modules():
            if isinstance(m, PackedModule) and m is not model.position_net:
                m.pk()
        # warm-up on a side stream (first-call attribute setup etc.), then capture
        with ops.capture_workspace(self.x.device):  # stream-K scratch of captured GEMMs, allocated up front
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                model._core(self.x, self.t, self.ctx, M, self.okv, n_obj, self.mask, self.scale, self.conv)
            torch.cuda.current_stream().wait_stream(s)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, pool=model.graph_pool):
                self.out = model._core(self.x, self.t, self.ctx, M, self.okv, n_obj, self.mask, self.scale, self.conv)

    def replay(self, x, t, ctx, okv, mask=None, fuser_scale=None, n_restored=None):
        self.x.copy_(x)
        self.t.copy_(t)
        if isinstance(self.scale, torch.Tensor):
            self.scale.copy_(fuser_scale)
        if isinstance(self.conv, torch.Tensor):
            self.conv.copy_(n_restored)
        # step-invariant inputs: the static buffers already hold them when the very same (immutable, cached)
        # tensor objects come back -- every step of a sampling run after the first
        last = getattr(self, "_last", (None, None, None))
        if ctx is not last[0]:
            self.ctx.copy_(ctx)
        if self.okv is not None and okv is not last[1]:
            for dst, src in zip(self.okv, okv):
                dst.copy_(src)
        if self.mask is not None and mask is not last[2]:
            self.mask[0].copy_(mask[0])
            self.mask[1].copy_(mask[1])
        self._last = (ctx, okv, mask)  # (references keep the identities unique)
        self.graph.replay()
        return self.out.clone()
