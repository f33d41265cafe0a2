"""`-m gpu` tests of continuous batching: the per-image input conv kernel (idiff_conv_in_select) against torch,
UNetModel.forward_batched(per_image_conv=True) against separate forwards, and SamplingEngine with staggered arrivals
against each request's own sampler run -- plus the graph bound, memory over repeated traces, two latent sizes at once
and one request anchored to the reference's golden latent."""
import os
import sys
from functools import partial

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
from test_requests_gpu import EPS_TOL, LATENT_TOL, _att_masks, _fresh, _rel, _reset, _run_alone  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")
BUCKETS = (2, 4, 8)


@pytest.fixture(scope="module")
def unet(cuda_device):
    from instancediffusion_b200.weights import build_unet
    model = build_unet("box", cuda_device, seed=0)
    model._sd_conv = torch.load(os.path.join(GOLDEN, "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(model._sd_conv))
    model.restore_first_conv_from_SD()  # the SD1.5 weights are known from here on
    model.undo_first_conv_restore()
    yield model
    model.use_cuda_graph = True


@pytest.fixture(scope="module")
def diffusion(cuda_device):
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)


# ------------------------------------------------------------------------------------------------
# 1. kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W", [(5, 64, 48), (3, 24, 40)])
def test_conv_in_select_matches_conv2d(cuda_device, dtype, B, H, W):
    from instancediffusion_b200 import ops
    from instancediffusion_b200.packing import pack_conv3x3_taps
    g = torch.Generator(device="cpu").manual_seed(B * H + W)
    x = torch.randn((B, 4, H, W), generator=g).to(cuda_device) * 2
    ws = [(torch.randn((320, 4, 3, 3), generator=g) * 0.2).to(cuda_device) for _ in range(2)]
    bs = [(torch.randn((320,), generator=g) * 0.1).to(cuda_device) for _ in range(2)]
    flags = torch.tensor([1, 0, 1, 1, 0][:B], dtype=torch.int32, device=cuda_device)
    with ops.storage(dtype):
        w16 = [w.to(dtype) for w in ws]
        out = ops.conv_in_select(x, pack_conv3x3_taps(w16[0]), bs[0], pack_conv3x3_taps(w16[1]), bs[1], flags)
        assert out.dtype == dtype and tuple(out.shape) == (B * H * W, 320)
    xr = x.to(dtype).float()  # the storage-rounded operands, in fp32
    for b in range(B):
        s = int(flags[b])
        ref = torch.nn.functional.conv2d(xr[b:b + 1], w16[s].float(), bs[s], padding=1)
        got = out.view(B, H, W, 320)[b].permute(2, 0, 1).float()
        r = _rel(got, ref[0])
        assert r < (1e-3 if dtype == torch.float16 else 6e-3), (b, r)


# ------------------------------------------------------------------------------------------------
# 2. forward_batched(per_image_conv=True)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True])
def test_forward_batched_per_image_conv(cuda_device, unet, graph):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.utils.model import set_alpha_scale
    gti = unet.grounding_tokenizer_input
    ia, uca = synthetic.make_sampler_inputs(gti, 1, 2, 171, "box", device=cuda_device)
    ib, _ = synthetic.make_sampler_inputs(gti, 1, 3, 172, "box", device=cuda_device)
    ts = [torch.full((1,), t, dtype=torch.long, device=cuda_device) for t in (601, 801, 401, 201)]
    inputs = [dict(x=ia["x"], timesteps=ts[0], context=ia["context"], grounding_input=ia["grounding_input"]),
              dict(x=ia["x"], timesteps=ts[1], context=uca),
              dict(x=ib["x"], timesteps=ts[2], context=ib["context"], grounding_input=ib["grounding_input"]),
              dict(x=ib["x"] * 0.5, timesteps=ts[3], context=ib["context"], grounding_input=ib["grounding_input"])]
    scales, restored = [1.0, 0.0, 0.5, 1.0], [True, False, True, False]
    unet.use_cuda_graph = graph
    try:
        _reset(unet)
        refs = []
        for inp, s, r in zip(inputs, scales, restored):
            set_alpha_scale(unet, s)
            if r:
                unet.restore_first_conv_from_SD()
            refs.append(unet(dict(inp)).clone())
            unet.undo_first_conv_restore()
        set_alpha_scale(unet, 1)
        for flags in (restored, [not r for r in restored]):  # a new flag pattern replays the same graph
            n = len(unet._graphs)
            got = unet.forward_batched(inputs, scales=scales, restored=flags, per_image_conv=True)
            assert not unet._first_conv_restored
            if flags is restored:
                for k, (g, ref) in enumerate(zip(got, refs)):
                    r = _rel(g, ref)
                    print(f"[per_image_conv graph={graph}] input {k}: rel_l2 {r:.2e}")
                    assert r < EPS_TOL, (k, r)
            else:
                assert len(unet._graphs) == n
    finally:
        _reset(unet)
        unet.use_cuda_graph = True


# ------------------------------------------------------------------------------------------------
# 3. SamplingEngine
# ------------------------------------------------------------------------------------------------
def _requests(unet, device):
    """Five requests: S in {10, 11, 20}; MIS 0.36 (one with the instance-isolation mask), MIS 1, plain PLMS, and one
    without an alpha schedule."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    out = []
    for seed, n, S, mis, alpha in ((201, 2, 10, 0.36, agen), (202, 2, 11, 0.0, agen), (203, 1, 20, 1.0, agen),
                                   (204, 3, 11, 0.36, partial(alpha_generator, type=[0.5, 0.0, 0.5])),
                                   (205, 4, 10, 0.0, None)):
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, n, seed, "box", mis=mis > 0, device=device)
        if seed == 201:
            for inp in inputs:
                inp["grounding_input"]["att_masks"] = _att_masks(inp["grounding_input"])
        out.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=alpha, mis=mis,
                           shape=(1, 4, 64, 64), S=S))
    return out


def _drive(engine, reqs, ticks):
    """Submit reqs[j] at tick ticks[j]; tick until all finished.  {j: latent}."""
    by_ticket, done, tick = {}, {}, 0
    while len(done) < len(reqs):
        for j, t in enumerate(ticks):
            if t == tick:
                by_ticket[engine.submit(_fresh(reqs[j]))] = j
        for ticket, x in engine.step().items():
            done[by_ticket[ticket]] = x
        tick += 1
    return done


def _graph_groups(keys):
    """Engine graph keys grouped by everything but the batch: (latent size, context length, fuser state, n_obj,
    mask presence, conv) -> batch sizes."""
    groups = {}
    for shape, M, scales, n_obj, mask, conv in keys:
        state = "off" if scales == () else ("per-image" if scales == ("per-image",) else "scalar")
        groups.setdefault((shape[1:], M, state, scales, n_obj, mask, conv), set()).add(shape[0])
    return groups


@pytest.mark.parametrize("graph", [False, True])
def test_engine_staggered_requests_match_their_own_samplers(cuda_device, unet, diffusion, graph):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = _requests(unet, cuda_device)
    alone = [_run_alone(unet, diffusion, r, r.S) for r in reqs]
    unet.use_cuda_graph = graph
    try:
        _reset(unet)
        before = set(unet._graphs)
        eng = SamplingEngine(unet, diffusion, max_batch=8, buckets=BUCKETS)
        got = _drive(eng, reqs, [0, 0, 3, 7, 12])
        assert eng.padded_images > 0 and eng.forwards > 0
        # the model is where it was: own conv, fuser scale 1
        assert not unet._first_conv_restored
        assert all(blk.fuser.scale == 1 for st in unet._transformers() for blk in st.transformer_blocks)
        for j, a in enumerate(alone):
            r = _rel(got[j], a)
            print(f"[engine graph={graph}] request {j} (S {reqs[j].S}, mis {reqs[j].mis}): rel_l2 vs alone {r:.2e}")
            assert r < LATENT_TOL, (j, r)
        if graph:
            new = set(unet._graphs) - before
            assert eng.graphs_captured == len(new) > 0
            for g, sizes in _graph_groups(new).items():
                assert sizes <= set(BUCKETS), (g, sizes)
            # another arrival pattern: every forward replays a graph already captured
            eng2 = SamplingEngine(unet, diffusion, max_batch=8, buckets=BUCKETS)
            got2 = _drive(eng2, reqs, [0, 2, 2, 5, 9])
            assert eng2.graphs_captured == 0
            for j, a in enumerate(alone):
                assert _rel(got2[j], a) < LATENT_TOL, j
        # without padding
        eng3 = SamplingEngine(unet, diffusion, max_batch=8, buckets=None)
        got3 = _drive(eng3, reqs, [0, 0, 3, 7, 12])
        assert eng3.padded_images == 0
        for j, a in enumerate(alone):
            r = _rel(got3[j], a)
            assert r < LATENT_TOL, (j, r)
    finally:
        _reset(unet)
        unet.use_cuda_graph = True


def test_engine_memory_is_bounded_over_repeated_traces(cuda_device, unet, diffusion):
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    reqs = _requests(unet, cuda_device)
    _reset(unet)
    try:
        used = []
        for _ in range(2):
            eng = SamplingEngine(unet, diffusion, max_batch=8, buckets=BUCKETS)
            _drive(eng, reqs, [0, 0, 3, 7, 12])
            torch.cuda.synchronize()
            used.append(torch.cuda.memory_allocated())
            # nothing of a finished request is left in the hoisted caches
            for r in reqs:
                for inp in (r.input if isinstance(r.input, list) else [r.input]):
                    assert unet._tkey(inp["context"]) not in unet._ctx_cache
                    assert unet._obj_key(inp["grounding_input"]) not in unet._obj_cache
                assert unet._tkey(r.uc) not in unet._ctx_cache
            assert len(unet._cat_cache) == 0
        print(f"[engine memory] allocated after each drain: {[u / 2**20 for u in used]} MiB")
        assert used[1] <= used[0] + 2 ** 20, used
    finally:
        _reset(unet)


def test_engine_reference_anchor_mid_run(cuda_device, unet, diffusion):
    """The samplers_extra mis_S10_n3 case (golden latent from the reference's own modules), submitted at tick 2 while
    two other requests run."""
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from instancediffusion_b200.utils.model import alpha_generator
    gold = torch.load(os.path.join(GOLDEN, "samplers_extra.pt"), map_location="cpu")
    sc = cases.SAMPLER_EXTRA_CASES["mis_S10_n3"]
    gti = unet.grounding_tokenizer_input
    others = _requests(unet, cuda_device)[1:3]
    inputs, uc = synthetic.make_sampler_inputs(gti, sc["batch"], sc["n"], sc["seed"], "box", mis=True, device=cuda_device)
    anchor = Request(input=inputs, uc=uc, guidance_scale=sc["guidance"], S=sc["S"],
                     alpha_generator_func=partial(alpha_generator, type=sc["alpha_type"]), mis=sc["mis"],
                     shape=(sc["batch"], 4, 64, 64))
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=BUCKETS), others + [anchor], [0, 1, 2])
    finally:
        _reset(unet)
    r = _rel(got[2], gold["mis_S10_n3"])
    print(f"[engine] mis_S10_n3 submitted mid-run: rel_l2 vs reference golden {r:.3e} (tol {LATENT_TOL:.1e})")
    assert r < LATENT_TOL, r


def test_engine_two_latent_sizes(cuda_device, unet, diffusion):
    from instancediffusion_b200 import synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from instancediffusion_b200.utils.model import alpha_generator
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    reqs = []
    for seed, size, mis in ((211, 64, 0.36), (212, 48, 0.36), (213, 48, 0.0)):
        inputs, uc = synthetic.make_sampler_inputs(gti, 1, 2, seed, "box", mis=mis > 0, device=cuda_device, size=size)
        reqs.append(Request(input=inputs, uc=uc, guidance_scale=7.5, alpha_generator_func=agen, mis=mis,
                            shape=(1, 4, size, size), S=10))
    alone = [_run_alone(unet, diffusion, r, r.S) for r in reqs]
    _reset(unet)
    try:
        got = _drive(SamplingEngine(unet, diffusion, max_batch=8, buckets=BUCKETS), reqs, [0, 1, 1])
    finally:
        _reset(unet)
    for j, a in enumerate(alone):
        r = _rel(got[j], a)
        print(f"[engine] {reqs[j].shape[2]}x{reqs[j].shape[3]} request {j}: rel_l2 vs alone {r:.2e}")
        assert r < LATENT_TOL, (j, r)
