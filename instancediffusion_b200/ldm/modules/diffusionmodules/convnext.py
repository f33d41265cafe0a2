"""ConvNeXt-tiny mask encoder inside UniFusion -- drop-in for ldm/modules/diffusionmodules/convnext.py
(:15-123: depths 3-3-9-3, dims 96/192/384/768; the same 178 state_dict keys, so reference checkpoints
load strict).  It only runs when a sample carries non-zero `segs` (mask conditioning,
text_grounding_net.py:226-231), once per sample after hoisting.

H100 mapping (activations NHWC fp16 == token-major rows):
  * stem Conv2d(3, 96, 4, stride 4) and the three Conv2d(C, 2C, 2, stride 2) downsamplers are
    kernel == stride convolutions: one coalesced patch gather (idiff_patchify) + a wgmma GEMM;
  * Block = depthwise 7x7 (idiff_dwconv7x7) -> LayerNorm over channels (idiff_layernorm; with NHWC rows the
    reference's permutes vanish) -> pwconv1 GEMM with the exact-erf GELU fused in the epilogue ->
    pwconv2 GEMM whose epilogue adds the block input; the layer-scale `gamma` is folded into pwconv2's
    weight and bias at pack time (gamma * (W h + b) = (diag(gamma) W) h + gamma * b, exact in real arithmetic);
  * the channels_first LayerNorms of the stem / downsamplers normalise over C per pixel, which is the same
    row LayerNorm in NHWC.
"""
import torch
import torch.nn as nn

from .... import ops
from .._base import half, PackedModule, f32, nchw_to_nhwc16, nhwc16_to_nchw, w16


class LayerNorm(nn.Module):
    """convnext.py:120-145 (parameter holder; both data formats are a per-pixel LayerNorm over C here)."""

    def __init__(self, normalized_shape, eps=1e-6, data_format="channels_last"):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps
        self.data_format = data_format
        if self.data_format not in ["channels_last", "channels_first"]:
            raise NotImplementedError
        self.normalized_shape = (normalized_shape,)


class Block(PackedModule):
    """convnext.py:15-51."""

    def __init__(self, dim, drop_path=0., layer_scale_init_value=1e-6):
        super().__init__()
        self.dim = dim
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, 4 * dim)
        self.pwconv2 = nn.Linear(4 * dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones((dim)), requires_grad=True) \
            if layer_scale_init_value > 0 else None

    def _pack(self):
        g = f32(self.gamma) if self.gamma is not None else None
        w2 = self.pwconv2.weight.detach().float()
        b2 = self.pwconv2.bias.detach().float()
        if g is not None:
            w2 = g[:, None] * w2
            b2 = g * b2
        return {
            # (C,1,7,7) -> [49][C] tap-major fp32
            "wd": self.dwconv.weight.detach().float().reshape(self.dim, 49).t().contiguous(),
            "bd": f32(self.dwconv.bias),
            "ng": f32(self.norm.weight), "nb": f32(self.norm.bias),
            "w1": w16(self.pwconv1.weight), "b1": f32(self.pwconv1.bias),
            "w2": w2.to(half()).contiguous(), "b2": b2.contiguous(),
        }

    def _fwd(self, x16, B, H, W):
        """x16 fp16 [B*H*W, C] -> same shape (new tensor)."""
        p = self.pk()
        h = ops.dwconv7x7(x16, p["wd"], p["bd"], B, H, W)
        h = ops.layernorm(h, p["ng"], p["nb"], self.norm.eps)
        h = ops.gemm(h, p["w1"], p["b1"], gelu=True)
        return ops.gemm(h, p["w2"], p["b2"], residual=x16)

    def forward(self, x):
        x16, B, H, W = nchw_to_nhwc16(x)
        return nhwc16_to_nchw(self._fwd(x16, B, H, W), B, H, W, x.dtype)


class ConvNeXt(PackedModule):
    """convnext.py:53-118 (no classifier head: UniFusion uses forward_features only)."""

    def __init__(self, in_chans=3, num_classes=1000, depths=(3, 3, 9, 3), dims=(96, 192, 384, 768),
                 drop_path_rate=0., layer_scale_init_value=1e-6, head_init_scale=1.):
        super().__init__()
        self.dims = list(dims)
        self.downsample_layers = nn.ModuleList()
        self.downsample_layers.append(nn.Sequential(
            nn.Conv2d(in_chans, dims[0], kernel_size=4, stride=4),
            LayerNorm(dims[0], eps=1e-6, data_format="channels_first")))
        for i in range(3):
            self.downsample_layers.append(nn.Sequential(
                LayerNorm(dims[i], eps=1e-6, data_format="channels_first"),
                nn.Conv2d(dims[i], dims[i + 1], kernel_size=2, stride=2)))
        self.stages = nn.ModuleList([
            nn.Sequential(*[Block(dim=dims[i], layer_scale_init_value=layer_scale_init_value) for _ in range(depths[i])])
            for i in range(4)])

    @staticmethod
    def _pack_patch_conv(conv: nn.Conv2d):
        """(Cout, Cin, p, p) -> [Cout, p*p*Cin] with k = (ky*p + kx)*Cin + c (idiff_patchify's column order)."""
        w = conv.weight.detach()
        return w16(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)), f32(conv.bias)

    def _pack(self):
        stem_conv, stem_ln = self.downsample_layers[0][0], self.downsample_layers[0][1]
        p = {"stem": self._pack_patch_conv(stem_conv) + (f32(stem_ln.weight), f32(stem_ln.bias), stem_ln.eps),
             "down": []}
        for i in range(1, 4):
            ln, conv = self.downsample_layers[i][0], self.downsample_layers[i][1]
            p["down"].append((f32(ln.weight), f32(ln.bias), ln.eps) + self._pack_patch_conv(conv))
        return p

    def _features(self, x16, B, H, W):
        """x16: fp16 NHWC [B*H*W, in_chans] -> (fp16 [B*(H/32)*(W/32), 768], H/32, W/32)."""
        p = self.pk()
        w, b, g, beta, eps = p["stem"]
        cin = x16.shape[-1]
        h = ops.gemm(ops.patchify(x16, B, H, W, cin, 4), w, b)
        H, W = H // 4, W // 4
        h = ops.layernorm(h, g, beta, eps)
        for i in range(4):
            if i > 0:
                g, beta, eps, w, b = p["down"][i - 1]
                h = ops.layernorm(h, g, beta, eps)
                h = ops.gemm(ops.patchify(h, B, H, W, self.dims[i - 1], 2), w, b)
                H, W = H // 2, W // 2
            for blk in self.stages[i]:
                h = blk._fwd(h, B, H, W)
        return h, H, W

    def forward_features(self, x):
        x16, B, H, W = nchw_to_nhwc16(x)
        h, Ho, Wo = self._features(x16, B, H, W)
        return nhwc16_to_nchw(h, B, Ho, Wo, x.dtype)

    def forward(self, x):
        return self.forward_features(x)


def convnext_tiny(pretrained=False, in_22k=False, **kwargs):
    """No network download here (the reference fetches ImageNet weights at construction,
    convnext.py:152-158); weights arrive with the InstanceDiffusion checkpoint."""
    return ConvNeXt(depths=[3, 3, 9, 3], dims=[96, 192, 384, 768], **kwargs)
