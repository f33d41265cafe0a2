"""UniFusion instance tokenizer -- drop-in for ldm/modules/diffusionmodules/text_grounding_net.py.

(box | point | scribble | polygon) Fourier embeddings + the CLIP phrase feature -> four 3-layer
MLPs, plus 64 mask tokens -> a fifth MLP; padded / dropped slots take learned null features.
Output (B, 30*4 + 64 = 184, 768) and `drop_box_mask`.

H100 mapping: one coalesced kernel per modality builds the MLP input matrix (Fourier embedding,
null substitution and the text concat fused, idiff_fourier_embed); the MLPs are weight-streaming
wgmma GEMMs with SiLU epilogues.  The result depends only on the sample's conditioning, so the
UNet calls this once per sample, not once per forward (text_grounding_net.py is re-run on every
forward in the reference, openaimodel.py:494).
"""
import torch
import torch.nn as nn

from .... import ops
from .._base import half, PackedModule, f32, w16
from .convnext import convnext_tiny
from .util import FourierEmbedder


class UniFusion(PackedModule):
    def __init__(self, in_dim, out_dim, mid_dim=3072, fourier_freqs=8,
                 train_add_boxes=True, train_add_points=True, train_add_scribbles=True, train_add_masks=True,
                 test_drop_boxes=False, test_drop_points=False, test_drop_scribbles=True, test_drop_masks=False,
                 use_seperate_tokenizer=True):
        super().__init__()
        if not (train_add_boxes and train_add_points and train_add_scribbles and train_add_masks
                and use_seperate_tokenizer):
            raise NotImplementedError("UniFusion: only the released configuration (all modalities, separate "
                                      "tokenizers) is supported")
        self.in_dim = in_dim
        self.out_dim = out_dim
        self.mid_dim = mid_dim
        self.n_scribble_points = 20
        self.n_polygon_points = 256
        fourier_freqs = 16  # hard-coded in the reference (:20-21) regardless of the ctor argument
        self.add_boxes = self.add_points = self.add_scribbles = self.add_masks = True
        self.use_seperate_tokenizer = True
        self.use_segs = True
        self.resize_input = 512
        self.down_factor = 64
        self.in_conv = nn.Conv2d(30, 3, 3, 1, 1)
        self.convnext_tiny_backbone = convnext_tiny(pretrained=True)
        self.num_tokens = (self.resize_input // self.down_factor) ** 2
        self.convnext_feature_dim = 3072
        self.pos_embedding = nn.Parameter(torch.empty(1, self.num_tokens, self.convnext_feature_dim).normal_(std=0.02))
        self.test_drop_boxes = test_drop_boxes
        self.test_drop_points = test_drop_points
        self.test_drop_scribbles = test_drop_scribbles
        self.test_drop_masks = test_drop_masks
        self.test_drop_segs = test_drop_masks
        self.fourier_embedder = FourierEmbedder(num_freqs=fourier_freqs)
        self.fourier_embedder_polygons = FourierEmbedder(num_freqs=fourier_freqs)
        self.position_dim = fourier_freqs * 2 * 4
        self.point_dim = fourier_freqs * 2 * 2
        self.scribble_dim = fourier_freqs * 2 * self.n_scribble_points * 2
        self.polygon_dim = fourier_freqs * 2 * self.n_polygon_points * 2
        dims = [in_dim + self.position_dim, in_dim + self.point_dim, in_dim + self.scribble_dim,
                in_dim + self.polygon_dim, self.convnext_feature_dim]
        self.linears_list = nn.ModuleList([
            nn.Sequential(nn.Linear(d, mid_dim), nn.SiLU(), nn.Linear(mid_dim, mid_dim), nn.SiLU(),
                          nn.Linear(mid_dim, out_dim)) for d in dims])
        self.null_positive_feature = nn.Parameter(torch.zeros([in_dim]))
        self.null_position_feature = nn.Parameter(torch.zeros([self.position_dim]))
        self.null_point_feature = nn.Parameter(torch.zeros([self.point_dim]))
        self.null_scribble_feature = nn.Parameter(torch.zeros([self.scribble_dim]))
        self.null_polygon_feature = nn.Parameter(torch.zeros([self.polygon_dim]))
        self.null_seg_feature = nn.Parameter(torch.zeros([self.convnext_feature_dim]))

    def reset_dropout_test(self):
        """text_grounding_net.py:105-117: (drop_point, drop_box, drop_scribble, drop_polygons, drop_segs)."""
        return (self.test_drop_points, self.test_drop_boxes, self.test_drop_scribbles,
                self.test_drop_masks, self.test_drop_masks)

    def _pack(self):
        p = {"mlp": []}
        for seq in self.linears_list:
            p["mlp"].append([(w16(seq[i].weight), f32(seq[i].bias)) for i in (0, 2, 4)])
        p["null_text"] = f32(self.null_positive_feature)
        p["null_box"] = f32(self.null_position_feature)
        p["null_point"] = f32(self.null_point_feature)
        p["null_scribble"] = f32(self.null_scribble_feature)
        p["null_polygon"] = f32(self.null_polygon_feature)
        # null seg tokens (segs all zero / dropped): null_seg + pos_embedding (:279-285), 64 rows
        p["seg_null_in"] = (f32(self.null_seg_feature)[None, :] + f32(self.pos_embedding)[0]).to(half()).contiguous()
        p["pos"] = f32(self.pos_embedding)[0].contiguous()
        p["w_inconv"] = f32(self.in_conv.weight)
        p["b_inconv"] = f32(self.in_conv.bias)
        return p

    @staticmethod
    def _all_planes_empty(segs: torch.Tensor) -> bool:
        """Cheap exact shortcut for the spatially-constant `segs` the null / box-only inputs carry
        (GroundingNetInput.get_null_input and synthetic.make_grounding_batch hand back a (B, N, 1, 1) tensor
        expanded over the spatial dims): with stride-0 planes, sum(segs[b]) > 0 iff sum_n segs[b, n, 0, 0] > 0,
        a B x N reduction.  Dense masks are never inspected on the host -- the kernels decide per sample."""
        if segs.dim() != 4 or segs.stride(-1) != 0 or segs.stride(-2) != 0:
            return False
        return not bool((segs[:, :, 0, 0].float().sum(dim=1) > 0).any())

    def _mlp(self, idx, x16):
        (w0, b0), (w1, b1), (w2, b2) = self.pk()["mlp"][idx]
        h = ops.gemm(x16, w0, b0, silu=True)
        h = ops.gemm(h, w1, b1, silu=True)
        return ops.gemm(h, w2, b2)

    @torch.no_grad()
    def _tokens(self, boxes, masks, positive_embeddings, scribbles=None, polygons=None, segs=None, points=None):
        """-> (objs fp16 [B*184, out_dim], B, 184, drop_box_mask)."""
        if self.training:
            raise NotImplementedError("UniFusion training-time modality dropout is out of scope (sampling path only)")
        p = self.pk()
        dev = p["null_text"].device
        B, N, _ = boxes.shape
        rows = B * N
        drop_point, drop_box, drop_scribble, drop_polygons, drop_segs = self.reset_dropout_test()
        if drop_point and drop_box and drop_scribble and drop_polygons and drop_segs:
            drop_box = False
        f = lambda t, d: t.to(device=dev, dtype=torch.float32).reshape(rows, d).contiguous()
        m = masks.to(device=dev, dtype=torch.float32).reshape(rows).contiguous()
        text = f(positive_embeddings, self.in_dim)
        if points is None:  # :219-220, a point can always be derived from a box
            points = (boxes[:, :, :2] + boxes[:, :, 2:]) / 2.0
        specs = [
            (f(boxes, 4), p["null_box"], 0, drop_box),
            (f(points, 2), p["null_point"], 0, drop_point),
            (f(scribbles, scribbles.shape[-1]), p["null_scribble"], 1, drop_scribble),
            (f(polygons, polygons.shape[-1]), p["null_polygon"], 1, drop_polygons),
        ]
        toks = []
        for idx, (coords, null_pos, mode, dropped) in enumerate(specs):
            D = coords.shape[1]
            if 32 * D != null_pos.numel():
                raise ValueError(f"UniFusion: modality {idx} expects {null_pos.numel() // 32} coordinates, got {D}")
            buf = torch.empty((rows, self.in_dim + 32 * D), dtype=half(), device=dev)
            ops.fourier_embed(coords, m, null_pos, buf, text=text, null_text=p["null_text"], mask_mode=mode,
                              dropped=dropped)
            toks.append(self._mlp(idx, buf).view(B, N, self.out_dim))
        # mask tokens (text_grounding_net.py:226-231, 277-287): ConvNeXt features of the resized binary masks,
        # reinterpreted as 64 tokens of 3072 features; samples whose masks sum to zero (and the dropped /
        # CFG-null case) take the learned null feature -- decided per sample on the device from the sum the
        # in_conv kernel accumulates.
        if not drop_segs and segs is not None and not self._all_planes_empty(segs):
            segs = segs.to(device=dev, dtype=torch.float32)
            y, seg_sum = ops.segs_inconv(segs, p["w_inconv"], p["b_inconv"], self.resize_input)
            feat, fh, fw = self.convnext_tiny_backbone._features(y, B, self.resize_input, self.resize_input)
            if fh * fw * feat.shape[-1] != self.num_tokens * self.convnext_feature_dim:
                raise ValueError("UniFusion: ConvNeXt feature map does not match num_tokens x convnext_feature_dim")
            seg_in = ops.seg_tokens(feat, p["seg_null_in"], p["pos"], seg_sum, B, fh * fw, self.num_tokens)
            seg_tok = self._mlp(4, seg_in).view(B, self.num_tokens, self.out_dim)
        else:
            seg_tok = self._mlp(4, p["seg_null_in"])  # [64, out_dim], identical for every sample
            seg_tok = seg_tok.view(1, self.num_tokens, self.out_dim).expand(B, self.num_tokens, self.out_dim)
        toks.append(seg_tok)
        objs = torch.cat(toks, dim=1).contiguous()
        drop_box_mask = True if drop_box and drop_polygons else False
        return objs.view(B * objs.shape[1], self.out_dim), B, objs.shape[1], drop_box_mask

    def forward(self, boxes, masks, positive_embeddings, scribbles=None, polygons=None, segs=None, points=None):
        objs16, B, n, drop_box_mask = self._tokens(boxes, masks, positive_embeddings, scribbles, polygons, segs, points)
        return objs16.view(B, n, self.out_dim).to(positive_embeddings.dtype), drop_box_mask
