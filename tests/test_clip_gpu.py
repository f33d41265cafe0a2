"""`-m gpu` tests of the CLIP text encoder on the H100 kernels (host prep, SURVEY.md section 8f-3): the two small kernels
against torch, the whole text tower against the golden produced by transformers' CLIPTextModel (the third-party model
the reference calls at ldm/modules/encoders/modules.py:147-165 and utils/model.py:146-151), the FrozenCLIPEmbedder /
get_clip_feature surface, and the bf16 build."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")

# bounds: about 2x the measured text-tower errors
CLIP_TOL = 2.4e-3


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape and torch.isfinite(a).all()
    return ((a - b).norm() / b.norm()).item()


def _sd(prefix=""):
    from instancediffusion_b200.ldm.modules.encoders.modules import CLIPTextModel
    from instancediffusion_b200.weights import synth_tensor
    with torch.device("meta"):
        m = CLIPTextModel()
    return {prefix + k: synth_tensor("clip." + k, tuple(v.shape), cases.WEIGHT_SEED) for k, v in m.state_dict().items()}


def test_embed_tokens(cuda_device):
    from instancediffusion_b200 import ops
    g = torch.Generator().manual_seed(1)
    tok = (torch.randn((1000, 768), generator=g) * 0.05).to(cuda_device).half()
    pos = (torch.randn((77, 768), generator=g) * 0.05).to(cuda_device).half()
    ids = torch.randint(0, 1000, (3, 77), generator=g).to(cuda_device)
    out = ops.embed_tokens(ids, tok, pos)
    ref = (tok.float()[ids] + pos.float()[None]).reshape(3 * 77, 768)
    assert (out.float() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()  # one fp16 rounding of the sum


@pytest.mark.parametrize("B,T,lens", [(3, 77, None), (2, 16, None), (3, 77, (4, 77, 30)), (1, 128, None)])
def test_causal_attention_small(cuda_device, B, T, lens):
    from instancediffusion_b200 import ops
    H, d = 12, 64
    g = torch.Generator().manual_seed(2)
    qkv = torch.randn((B * T, 3 * H * d), generator=g).to(cuda_device).half()
    kl = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=cuda_device)
    out = ops.causal_attention_small(qkv, batch=B, tokens=T, heads=H, head_dim=d, scale=d ** -0.5, key_len=kl)
    q, k, v = [t.float().view(B, T, H, d).transpose(1, 2) for t in qkv.split(H * d, dim=1)]
    mask = torch.full((T, T), float("-inf"), device=cuda_device).triu(1)[None, None].expand(B, 1, T, T).clone()
    if lens is not None:
        for b, n in enumerate(lens):
            mask[b, :, :, n:] = float("-inf")
    ref = (torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5 + mask, dim=-1) @ v).transpose(1, 2).reshape(B * T, H * d)
    got = out.float()
    if lens is not None:  # rows whose every key is masked do not exist here (key 0 is always visible: len >= 1)
        assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item()
    print(f"[causal_attention_small B{B} T{T} lens={lens}] max_abs_err={err:.3e} ref_max={ref.abs().max().item():.3e}")
    assert err < 2e-3 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("name", list(cases.CLIP_CASES))
def test_clip_text_tower_vs_transformers_golden(cuda_device, name):
    from instancediffusion_b200.ldm.modules.encoders.modules import CLIPTextModel
    gold = torch.load(os.path.join(GOLDEN, "clip_text.pt"), map_location="cpu")
    m = CLIPTextModel()
    m.load_state_dict(_sd(), strict=True)
    m = m.to(cuda_device).eval()
    ids = cases.clip_token_ids(cases.CLIP_CASES[name]).to(cuda_device)
    out = m(input_ids=ids)
    r_last = _rel(out.last_hidden_state, gold[name + "/last_hidden_state"])
    r_pool = _rel(out.pooler_output, gold[name + "/pooler_output"])
    print(f"[clip/{name}] rel_l2 last_hidden_state {r_last:.3e} pooler_output {r_pool:.3e} (tol {CLIP_TOL:.0e})")
    assert r_last < CLIP_TOL and r_pool < CLIP_TOL


def test_frozen_clip_embedder_surface(cuda_device):
    """The reference's `text_encoder` checkpoint entry (keys `transformer.text_model...`, incl. the position_ids buffer
    transformers 4.27 saved) loads strict; forward takes token ids when no tokenizer files exist; get_clip_feature
    returns the pooled feature of the same tower."""
    from instancediffusion_b200.ldm.modules.encoders.modules import FrozenCLIPEmbedder, get_clip_feature
    gold = torch.load(os.path.join(GOLDEN, "clip_text.pt"), map_location="cpu")
    enc = FrozenCLIPEmbedder(device=cuda_device)
    sd = _sd("transformer.")
    sd["transformer.text_model.embeddings.position_ids"] = torch.arange(77).unsqueeze(0)
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(cuda_device)
    ids = cases.clip_token_ids(cases.CLIP_CASES["clip_b3"])
    z, pooled = enc.encode(ids, return_pooler_output=True)
    assert tuple(z.shape) == (3, 77, 768) and tuple(pooled.shape) == (3, 768)
    assert _rel(z, gold["clip_b3/last_hidden_state"]) < CLIP_TOL
    one = get_clip_feature(enc.transformer, None, ids[1:2])
    assert _rel(one, gold["clip_b3/pooler_output"][1:2]) < CLIP_TOL
    if enc.tokenizer is None:
        with pytest.raises(RuntimeError):
            enc("a photo of a cat")


def test_clip_text_tower_bf16(cuda_device):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.modules.encoders.modules import CLIPTextModel
    gold = torch.load(os.path.join(GOLDEN, "clip_text.pt"), map_location="cpu")
    with ops.storage(torch.bfloat16):
        m = CLIPTextModel()
        m.load_state_dict(_sd(), strict=True)
        m = m.to(cuda_device).eval()
        out = m(input_ids=cases.clip_token_ids(cases.CLIP_CASES["clip_b3"]).to(cuda_device))
        r = _rel(out.last_hidden_state, gold["clip_b3/last_hidden_state"])
    print(f"[clip bf16] rel_l2 last_hidden_state {r:.3e} (tol {8 * CLIP_TOL:.0e})")
    assert r < 8 * CLIP_TOL
