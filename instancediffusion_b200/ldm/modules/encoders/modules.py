"""CLIP text encoder on the H100 kernels -- drop-in for the text side of ldm/modules/encoders/modules.py:144-172
(`FrozenCLIPEmbedder`: prompt -> (B, 77, 768) context, optionally the pooled feature) and for the phrase features
of utils/model.py:130-152 (`get_clip_feature`: `outputs.text_model_output.pooler_output` of the same text tower).

Both wrap Hugging Face `CLIPTextModel` ("openai/clip-vit-large-patch14": 12 layers, width 768, 12 heads of 64,
MLP 3072 with QuickGELU, causal mask, 77 positions; transformers 4.27 pinned by requirements.txt:247).  The classes
below keep its parameter names (`text_model.embeddings.token_embedding.weight`, `...encoder.layers.N.self_attn.q_proj.
weight`, ...), so the `text_encoder` entry of a reference checkpoint (utils/checkpoint.py:246, keys prefixed
`transformer.`) loads strict, and evaluate it with:

    idiff_embed_tokens                 token + position embeddings
    idiff_layernorm                    pre-LN of each block, final LN
    idiff_gemm                         fused QKV (bias), out-proj (+ residual), fc1 (SiLU epilogue), fc2 (+ residual)
    idiff_causal_attention_small       77-token causal attention, one CTA per (sequence, head)

QuickGELU(u) = u * sigmoid(1.702 u) runs as the GEMM's SiLU epilogue on fc1 weights / bias pre-scaled by 1.702, with
fc2's weights scaled by 1 / 1.702 (exact in real arithmetic).  The tokenizer is host string processing and stays the
reference's (`transformers.CLIPTokenizer`); without its vocabulary files (offline) pass token ids directly.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import torch
import torch.nn as nn

from .... import ops
from .._base import PackedModule, f32, w16

QUICK_GELU = 1.702


class AbstractEncoder(nn.Module):
    def encode(self, *args, **kwargs):
        raise NotImplementedError


class _Attn(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.k_proj = nn.Linear(width, width)
        self.v_proj = nn.Linear(width, width)
        self.q_proj = nn.Linear(width, width)
        self.out_proj = nn.Linear(width, width)


class _Mlp(nn.Module):
    def __init__(self, width, inner):
        super().__init__()
        self.fc1 = nn.Linear(width, inner)
        self.fc2 = nn.Linear(inner, width)


class _Layer(nn.Module):
    def __init__(self, width, inner):
        super().__init__()
        self.self_attn = _Attn(width)
        self.layer_norm1 = nn.LayerNorm(width)
        self.mlp = _Mlp(width, inner)
        self.layer_norm2 = nn.LayerNorm(width)


class _Encoder(nn.Module):
    def __init__(self, width, inner, layers):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(width, inner) for _ in range(layers)])


class _Embeddings(nn.Module):
    def __init__(self, vocab, width, positions):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, width)
        self.position_embedding = nn.Embedding(positions, width)
        # (transformers 4.27 saves this buffer; newer versions do not: accepted on load, never required)
        self.register_buffer("position_ids", torch.arange(positions).unsqueeze(0), persistent=False)

    def _load_from_state_dict(self, state_dict, prefix, *a, **k):
        state_dict.pop(prefix + "position_ids", None)
        return super()._load_from_state_dict(state_dict, prefix, *a, **k)


class CLIPTextTransformer(PackedModule):
    """`CLIPTextModel.text_model` (modeling_clip.CLIPTextTransformer): parameters in HF's layout, forward on the kernels."""

    def __init__(self, vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                 num_attention_heads=12, max_position_embeddings=77, layer_norm_eps=1e-5):
        super().__init__()
        self.width, self.heads, self.eps = hidden_size, num_attention_heads, layer_norm_eps
        self.embeddings = _Embeddings(vocab_size, hidden_size, max_position_embeddings)
        self.encoder = _Encoder(hidden_size, intermediate_size, num_hidden_layers)
        self.final_layer_norm = nn.LayerNorm(hidden_size)

    def _pack(self):
        p = {"tok": w16(self.embeddings.token_embedding.weight), "pos": w16(self.embeddings.position_embedding.weight),
             "gf": f32(self.final_layer_norm.weight), "bf": f32(self.final_layer_norm.bias), "layers": []}
        for lyr in self.encoder.layers:
            a, m = lyr.self_attn, lyr.mlp
            p["layers"].append({
                "g1": f32(lyr.layer_norm1.weight), "b1": f32(lyr.layer_norm1.bias),
                "wqkv": w16(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0)),
                "bqkv": f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0)),
                "wo": w16(a.out_proj.weight), "bo": f32(a.out_proj.bias),
                "g2": f32(lyr.layer_norm2.weight), "b2": f32(lyr.layer_norm2.bias),
                "w1": w16(m.fc1.weight.detach().float() * QUICK_GELU), "bb1": f32(m.fc1.bias.detach().float() * QUICK_GELU),
                "w2": w16(m.fc2.weight.detach().float() / QUICK_GELU), "bb2": f32(m.fc2.bias),
            })
        return p

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, key_len: Optional[torch.Tensor] = None):
        """input_ids int64 (B, T <= 77) on the GPU -> (last_hidden_state fp32 (B, T, C), pooler_output fp32 (B, C)).
        key_len (optional int32 (B,)): number of real tokens per sequence when a padded batch carries an attention
        mask (get_clip_feature passes the processor's; FrozenCLIPEmbedder passes none)."""
        p = self.pk()
        B, T = input_ids.shape
        C, H = self.width, self.heads
        d = C // H
        x = ops.embed_tokens(input_ids, p["tok"], p["pos"])
        for L in p["layers"]:
            h = ops.layernorm(x, L["g1"], L["b1"], self.eps)
            qkv = ops.gemm(h, L["wqkv"], L["bqkv"])
            att = ops.causal_attention_small(qkv, batch=B, tokens=T, heads=H, head_dim=d, scale=d ** -0.5, key_len=key_len)
            x = ops.gemm(att, L["wo"], L["bo"], residual=x)
            h = ops.layernorm(x, L["g2"], L["b2"], self.eps)
            u = ops.gemm(h, L["w1"], L["bb1"], silu=True)
            x = ops.gemm(u, L["w2"], L["bb2"], residual=x)
        last = ops.layernorm(x, p["gf"], p["bf"], self.eps).float().view(B, T, C)
        # modeling_clip (4.27): the pooled feature is the hidden state at the end-of-text token = the highest id
        pooled = last[torch.arange(B, device=last.device), input_ids.argmax(dim=-1)]
        return last, pooled


class CLIPTextModel(PackedModule):
    """Stand-in for transformers.CLIPTextModel: `.text_model`, `forward(input_ids=...)` -> object with
    `last_hidden_state` and `pooler_output`."""

    def __init__(self, **config):
        super().__init__()
        self.text_model = CLIPTextTransformer(**config)

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, **unused):
        key_len = None
        if attention_mask is not None:
            key_len = attention_mask.to(torch.int32).sum(dim=-1).to(torch.int32).contiguous()
        last, pooled = self.text_model(input_ids, key_len)
        return SimpleNamespace(last_hidden_state=last, pooler_output=pooled)


class FrozenCLIPEmbedder(AbstractEncoder):
    """ldm/modules/encoders/modules.py:144-172 with the text tower on the H100 kernels.  `tokenizer`: any callable with
    the CLIPTokenizer call signature; by default transformers.CLIPTokenizer.from_pretrained(version) is tried and, if
    its files are not available (offline), left None -- `forward` then accepts a LongTensor of token ids."""

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, tokenizer=None):
        super().__init__()
        if tokenizer is None:
            try:
                from transformers import CLIPTokenizer
                tokenizer = CLIPTokenizer.from_pretrained(version, local_files_only=True)
                if getattr(tokenizer, "vocab_size", 0) < 49408:  # (no vocabulary files: recent versions hand back a stub)
                    tokenizer = None
            except Exception:
                tokenizer = None
        self.tokenizer = tokenizer
        self.transformer = CLIPTextModel()
        self.device = device
        self.max_length = max_length
        self.freeze()

    def freeze(self):
        self.transformer = self.transformer.eval()
        for param in self.parameters():
            param.requires_grad = False

    @torch.no_grad()
    def forward(self, text, return_pooler_output=False):
        if torch.is_tensor(text):
            tokens = text.to(device=self.device, dtype=torch.long)
        else:
            if self.tokenizer is None:
                raise RuntimeError("FrozenCLIPEmbedder: no tokenizer (CLIPTokenizer files not available); pass one to the "
                                   "constructor or call with a LongTensor of token ids")
            enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                                 return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
            tokens = enc["input_ids"].to(self.device)
        out = self.transformer(input_ids=tokens)
        return (out.last_hidden_state, out.pooler_output) if return_pooler_output else out.last_hidden_state

    def encode(self, text, return_pooler_output=False):
        return self(text, return_pooler_output)


@torch.no_grad()
def get_clip_feature(model, processor, input, is_image=False):
    """utils/model.py:130-152 for text: the pooled feature of one phrase.  `model`: an object with `.text_model`
    (CLIPTextModel above, or FrozenCLIPEmbedder().transformer); `processor`: a callable returning `input_ids` (and
    optionally `attention_mask`) for a string, or None when `input` already is a LongTensor of token ids."""
    if input is None:
        return None
    if torch.is_tensor(input):
        ids, mask = input, None
    else:
        enc = processor(text=input, return_tensors="pt", padding=True)
        ids, mask = enc["input_ids"], enc.get("attention_mask")
    dev = next(model.parameters()).device
    out = model(input_ids=ids.to(dev), attention_mask=None if mask is None else mask.to(dev))
    return out.pooler_output
