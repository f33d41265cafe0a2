"""First-stage autoencoder blocks (SD1.5 VAE), same class names / constructor signatures / state_dict keys
as the reference's ldm/modules/diffusionmodules/model.py, with the arithmetic in libidiff_b200.so:

  ResnetBlock (model.py:82-141)  GroupNorm(eps 1e-6)+swish -> conv3x3 -> GroupNorm+swish -> conv3x3 (+ skip or
                                 1x1 nin_shortcut) : idiff_groupnorm + idiff_gemm (implicit-GEMM convolution,
                                 residual add in the epilogue)
  AttnBlock   (model.py:150-202) single-head attention over all pixels, head_dim = channels (512): fused
                                 q|k projection GEMM (1/sqrt(c) folded into q), scores = q k^T as one GEMM per
                                 image, idiff_softmax_rows, (P V) as a GEMM against V^T -- which is produced
                                 directly, transposed, by running the v projection as W_v . x^T (the v bias
                                 moves behind the softmax, whose rows sum to one, into the proj_out bias)
  Upsample / Downsample (42-76)  nearest 2x + conv3x3 ; F.pad(0,1,0,1) + stride-2 conv (im2col operand)
  Decoder (462-569) / Encoder (368-460); Encoder.forward_images runs conv_in on uint8 image bytes
                                 (idiff_encode_image_in) instead of a 64-channel padded copy and a conv GEMM

Internal convention as in the UNet: fp16 token-major activations [B*H*W, C] (== NHWC) from the first
convolution to the last; the decoder's image leaves as fp32 NCHW straight from the last GEMM's epilogue.
The reference runs this stage in fp32 outside autocast (inference.py:96); here it is fp16 storage with
fp32 accumulation / statistics, checked against the reference's fp32 output (tests/golden/vae.pt).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .... import ops
from ....packing import pack_conv1x1, pack_conv3x3, pack_conv3x3_taps
from .._base import half, PackedModule, f32, nchw_to_nhwc16, nhwc16_to_nchw, w16


def nonlinearity(x):
    return x * torch.sigmoid(x)  # swish (model.py:33-35); the kernels fuse it into the GroupNorm pass


def Normalize(in_channels, num_groups=32):
    return torch.nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def _pack3x3(conv: nn.Conv2d, cin_pad: int | None = None) -> torch.Tensor:
    w = conv.weight.detach().to(half())
    cout, cin = w.shape[:2]
    if cin_pad is not None and cin_pad != cin:
        wp = torch.zeros((cout, cin_pad, 3, 3), dtype=half(), device=w.device)
        wp[:, :cin] = w
        w = wp
    return pack_conv3x3(w.contiguous())


class Upsample(PackedModule):
    """model.py:42-57."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        self.in_channels = in_channels
        if self.with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        return {"w": _pack3x3(self.conv), "b": f32(self.conv.bias)} if self.with_conv else {}

    def _fwd(self, x16, B, H, W):
        up = ops.upsample_nearest2x(x16, B, H, W)
        if not self.with_conv:
            return up
        p = self.pk()
        return ops.gemm(up, p["w"], p["b"], conv=(B, 2 * H, 2 * W, self.in_channels))

    def forward(self, x):
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, 2 * H, 2 * W, x.dtype)


class Downsample(PackedModule):
    """model.py:60-79 (with_conv=True: asymmetric zero pad + stride-2 convolution)."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        self.in_channels = in_channels
        if not with_conv:
            raise NotImplementedError("Downsample(with_conv=False) (average pooling) is not used by the SD1.5 first stage")
        self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def _pack(self):
        return {"w": _pack3x3(self.conv), "b": f32(self.conv.bias)}

    def _fwd(self, x16, B, H, W):
        p = self.pk()
        return ops.gemm(ops.im2col_s2(x16, B, H, W, pad01=True), p["w"], p["b"])

    def forward(self, x):
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, H // 2, W // 2, x.dtype)


class ResnetBlock(PackedModule):
    """model.py:82-141 with temb_channels == 0 (the autoencoder has no timestep embedding)."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        if temb_channels > 0:
            raise NotImplementedError("ResnetBlock with a timestep embedding is not part of the first-stage model")
        self.norm1 = Normalize(in_channels)
        self.conv1 = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = Normalize(out_channels)
        self.dropout = torch.nn.Dropout(dropout)
        self.conv2 = torch.nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                self.conv_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
            else:
                self.nin_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def _pack(self):
        p = {
            "g1": f32(self.norm1.weight), "b1": f32(self.norm1.bias), "w1": _pack3x3(self.conv1), "cb1": f32(self.conv1.bias),
            "g2": f32(self.norm2.weight), "b2": f32(self.norm2.bias), "w2": _pack3x3(self.conv2), "cb2": f32(self.conv2.bias),
        }
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                p["ws"], p["bs"] = _pack3x3(self.conv_shortcut), f32(self.conv_shortcut.bias)
            else:
                p["ws"], p["bs"] = pack_conv1x1(w16(self.nin_shortcut.weight)), f32(self.nin_shortcut.bias)
        return p

    def _fwd(self, x16, B, H, W):
        p = self.pk()
        hw = H * W
        h = ops.groupnorm(x16, p["g1"], p["b1"], batch=B, hw=hw, groups=32, eps=1e-6, silu=True)
        h = ops.gemm(h, p["w1"], p["cb1"], conv=(B, H, W, self.in_channels))
        h = ops.groupnorm(h, p["g2"], p["b2"], batch=B, hw=hw, groups=32, eps=1e-6, silu=True)
        if "ws" not in p:
            skip = x16
        elif self.use_conv_shortcut:
            skip = ops.gemm(x16, p["ws"], p["bs"], conv=(B, H, W, self.in_channels))
        else:
            skip = ops.gemm(x16, p["ws"], p["bs"])
        return ops.gemm(h, p["w2"], p["cb2"], conv=(B, H, W, self.out_channels), residual=skip)

    def forward(self, x, temb=None):
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, H, W, x.dtype)


class AttnBlock(PackedModule):
    """model.py:150-202: x + proj_out(softmax(q k^T / sqrt(c)) v), one head over all H*W pixels."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)

    def _pack(self):
        c = self.in_channels
        s = float(int(c) ** (-0.5))
        wq = self.q.weight.detach().float().reshape(c, c) * s          # the score scale folded into q
        bq = self.q.bias.detach().float() * s
        wk = self.k.weight.detach().float().reshape(c, c)
        wo = self.proj_out.weight.detach().float().reshape(c, c)
        # softmax rows sum to one: P (V + 1 b_v^T) = P V + b_v^T, so the v bias is applied after the
        # attention as part of the output projection's bias
        bo = self.proj_out.bias.detach().float() + wo @ self.v.bias.detach().float()
        return {
            "g": f32(self.norm.weight), "b": f32(self.norm.bias),
            "wqk": torch.cat([wq, wk], 0).to(half()).contiguous(),
            "bqk": torch.cat([bq, self.k.bias.detach().float()], 0).contiguous(),
            "wv": pack_conv1x1(w16(self.v.weight)),
            "wo": wo.to(half()).contiguous(), "bo": bo.contiguous(),
        }

    def _fwd(self, x16, B, H, W):
        p = self.pk()
        c, n = self.in_channels, H * W
        hn = ops.groupnorm(x16, p["g"], p["b"], batch=B, hw=n, groups=32, eps=1e-6, silu=False)
        qk = ops.gemm(hn, p["wqk"], p["bqk"])                       # [B*n, 2c] = [q / sqrt(c) | k]
        att = torch.empty((B * n, c), dtype=half(), device=x16.device)
        scores = torch.empty((n, n), dtype=half(), device=x16.device)  # one image at a time (n = 4096: 32 MB)
        for b in range(B):
            rows = slice(b * n, (b + 1) * n)
            ops.gemm(qk[rows, :c], qk[rows, c:], out=scores)        # q k^T (A = q rows, "weights" = k rows)
            ops.softmax_rows_(scores)
            vt = ops.gemm(p["wv"], hn[rows])                        # W_v x^T = V^T [c, n] (bias: see _pack)
            ops.gemm(scores, vt, out=att[rows])                     # P V
        return ops.gemm(att, p["wo"], p["bo"], residual=x16)

    def forward(self, x):
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, H, W, x.dtype)


def make_attn(in_channels, attn_type="vanilla"):
    assert attn_type in ["vanilla", "linear", "none"], f'attn_type {attn_type} unknown'
    if attn_type == "vanilla":
        return AttnBlock(in_channels)
    if attn_type == "none":
        return nn.Identity(in_channels)
    raise NotImplementedError("LinAttnBlock is not used by the SD1.5 first stage (configs: attn_type vanilla)")


class _Level(nn.Module):
    """Plain attribute holder, like the reference's bare nn.Module() levels (state_dict key compatibility)."""


class Encoder(PackedModule):
    """model.py:368-460."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        if use_linear_attn:
            attn_type = "linear"
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.conv_in = torch.nn.Conv2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
        self.down = nn.ModuleList()
        for i_level in range(self.num_resolutions):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch,
                                         dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(make_attn(block_in, attn_type=attn_type))
            down = _Level()
            down.block = block
            down.attn = attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, kernel_size=3, stride=1,
                                        padding=1)

    def _pack(self):
        p = {
            "w_in": _pack3x3(self.conv_in, _pad64(self.in_channels)), "b_in": f32(self.conv_in.bias),
            "g_out": f32(self.norm_out.weight), "b_out": f32(self.norm_out.bias),
            "w_out": _pack3x3(self.conv_out), "cb_out": f32(self.conv_out.bias),
        }
        if self.in_channels == 3:
            p["w_img"] = pack_conv3x3_taps(self.conv_in.weight.detach().to(half()))
        return p

    @torch.no_grad()
    def forward(self, x):
        p = self.pk()
        B, _, H, W = x.shape
        h = ops.nchw_f32_to_nhwc_f16(x.float(), _pad64(self.in_channels))
        h = ops.gemm(h, p["w_in"], p["b_in"], conv=(B, H, W, _pad64(self.in_channels)))
        return self._encode_tokens(h, B, H, W)

    @torch.no_grad()
    def forward_images(self, images):
        """`forward` of uint8 RGB images (B, H, W, 3) on the device, normalised as the reference's data loader does
        (u / 127.5 - 1, dataset/decode_item.py:567-568): conv_in reads the bytes (ops.encode_image_in)."""
        if self.in_channels != 3:
            raise NotImplementedError(f"forward_images needs a 3-channel conv_in (in_channels={self.in_channels})")
        p = self.pk()
        B, H, W, _ = images.shape
        return self._encode_tokens(ops.encode_image_in(images, p["w_img"], p["b_in"]), B, H, W)

    def _encode_tokens(self, h, B, H, W):
        """conv_in's output tokens [B*H*W, ch] -> conv_out fp32 NCHW (B, 2*z_channels, H/8, W/8)."""
        p = self.pk()
        for i_level in range(self.num_resolutions):
            lvl = self.down[i_level]
            for i_block in range(self.num_res_blocks):
                h = lvl.block[i_block]._fwd(h, B, H, W)
                if len(lvl.attn) > 0:
                    h = lvl.attn[i_block]._fwd(h, B, H, W)
            if i_level != self.num_resolutions - 1:
                h = lvl.downsample._fwd(h, B, H, W)
                H, W = H // 2, W // 2
        h = self.mid.block_1._fwd(h, B, H, W)
        h = self.mid.attn_1._fwd(h, B, H, W)
        h = self.mid.block_2._fwd(h, B, H, W)
        h = ops.groupnorm(h, p["g_out"], p["b_out"], batch=B, hw=H * W, groups=32, eps=1e-6, silu=True)
        out = torch.empty((B, self.conv_out.out_channels, H, W), dtype=torch.float32, device=h.device)
        ops.gemm(h, p["w_out"], p["cb_out"], conv=(B, H, W, self.conv_out.in_channels), out_nchw=out)
        return out


class Decoder(PackedModule):
    """model.py:462-569.  `forward(z)` takes the (already post_quant_conv-ed) latent like the reference;
    AutoencoderKL.decode feeds `_decode_tokens` directly with the fused latent prologue."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if use_linear_attn:
            attn_type = "linear"
        if give_pre_end or tanh_out:
            raise NotImplementedError("Decoder(give_pre_end / tanh_out) are not used by the shipped configs")
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.give_pre_end = give_pre_end
        self.tanh_out = tanh_out
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.z_channels = z_channels
        self.conv_in = torch.nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = _Level()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch,
                                         dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(make_attn(block_in, attn_type=attn_type))
            up = _Level()
            up.block = block
            up.attn = attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)  # prepend to get consistent order
        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)

    def _pack(self):
        return {
            "w_in": _pack3x3(self.conv_in, _pad64(self.z_channels)), "b_in": f32(self.conv_in.bias),
            "g_out": f32(self.norm_out.weight), "b_out": f32(self.norm_out.bias),
            "w_out": _pack3x3(self.conv_out), "cb_out": f32(self.conv_out.bias),
        }

    def _decode_tokens(self, z16, B, H, W):
        """z16: fp16 NHWC latent [B*H*W, 64] (channels >= z_channels zero) -> image fp32 (B, out_ch, 8H, 8W)."""
        p = self.pk()
        h = ops.gemm(z16, p["w_in"], p["b_in"], conv=(B, H, W, _pad64(self.z_channels)))
        h = self.mid.block_1._fwd(h, B, H, W)
        h = self.mid.attn_1._fwd(h, B, H, W)
        h = self.mid.block_2._fwd(h, B, H, W)
        for i_level in reversed(range(self.num_resolutions)):
            lvl = self.up[i_level]
            for i_block in range(self.num_res_blocks + 1):
                h = lvl.block[i_block]._fwd(h, B, H, W)
                if len(lvl.attn) > 0:
                    h = lvl.attn[i_block]._fwd(h, B, H, W)
            if i_level != 0:
                h = lvl.upsample._fwd(h, B, H, W)
                H, W = 2 * H, 2 * W
        h = ops.groupnorm(h, p["g_out"], p["b_out"], batch=B, hw=H * W, groups=32, eps=1e-6, silu=True)
        out = torch.empty((B, self.conv_out.out_channels, H, W), dtype=torch.float32, device=z16.device)
        ops.gemm(h, p["w_out"], p["cb_out"], conv=(B, H, W, self.conv_out.in_channels), out_nchw=out)
        return out

    @torch.no_grad()
    def forward(self, z):
        B, _, H, W = z.shape
        self.last_z_shape = z.shape
        return self._decode_tokens(ops.nchw_f32_to_nhwc_f16(z.float(), _pad64(self.z_channels)), B, H, W)
