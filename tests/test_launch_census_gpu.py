"""`-m gpu` launch census: every kernel launch the model really makes -- UNet forwards at 64x64 (a mixed batch: cond
and uncond, the instance-isolation mask, fuser scales 1 / 0.36 / 0, the SD first conv restored on some images), at
96x96, at the bench's batch (4 + 4, 8 instances), in the mask flavour (the ConvNeXt mask encoder), one VAE decode to
512^2, and a short sample_requests run of four sampler kinds -- is recorded through the `ops` entry points in both
modes (batch-invariant on and off) and both storage types, deduplicated by launch signature (shapes, strides, flags,
epilogue options, mode, storage type), and replayed against a float64 reference of the same operation on the same
recorded inputs.  The references and the one bound per op are in tests/cases_census.py.  Any err / bound above 1, or
a non-finite output, fails; the worst ratio per signature and per op family is printed.

The producer LayerNorm statistics (want_stats) are checked slot by slot against float64 sums of the stored output's
columns: the tile width that ran is the one whose column partition the slots fit (printed per signature), so a slot
count that does not match ceil(N / BN) of that width fails too.
"""
import inspect
import math
import os
import sys
import time
from collections import defaultdict

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
import cases_census as CC  # noqa: E402
import cases_ddim as CD  # noqa: E402
import cases_dpm as CDP  # noqa: E402
import cases_img2img as CI  # noqa: E402
import cases_inpaint as CP  # noqa: E402
import cases_noise as CN  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden")

# ops.silu is not wrapped: only the module-level ResBlock forward calls it (the UNet fuses SiLU into a GEMM epilogue)
FORWARD_OPS = ("gemm", "attention", "groupnorm", "layernorm", "scaleu_concat", "conv_in_select", "im2col_s2",
               "upsample_nearest2x", "timestep_embedding", "row_stats", "softmax_rows_", "vae_latent_in",
               "nchw_f32_to_nhwc_f16", "fourier_embed", "segs_inconv", "patchify", "dwconv7x7", "seg_tokens")
SAMPLING_OPS = ("plms_update", "latent_mean", "ddim_update", "dpmpp2m_update", "noise_latent", "inpaint_blend")
# arguments a kernel writes (recorded after the call)
WRITTEN = {"plms_update": ("e_out", "x_out"), "ddim_update": ("e_out", "x_out"), "dpmpp2m_update": ("x0_out", "x_out")}
KEEP = 2  # records kept per signature
MODES = {"default": False, "invariant": True}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
E64 = 64 * CC.E32  # fp32 elementwise sampling updates: |y - y64| <= 64 e (|y64| + Mag)


def _clone(v):
    from instancediffusion_b200 import ops
    if isinstance(v, torch.Tensor):
        return v.clone()
    if isinstance(v, ops.RowStats):
        return ops.RowStats(v.t.clone(), v.slots)
    if isinstance(v, (list, tuple)):
        return type(v)(_clone(x) for x in v)
    return v


class Recorder:
    """Wraps ops entry points; keeps the first KEEP launches of every signature: (named inputs, output, written)."""

    def __init__(self, monkeypatch, names):
        from instancediffusion_b200 import ops
        self.records = defaultdict(list)
        for name in names:
            orig = getattr(ops, name)
            monkeypatch.setattr(ops, name, self._wrap(name, orig, inspect.signature(orig)))

    def _wrap(self, name, orig, sig):
        from instancediffusion_b200 import ops

        def wrapper(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            named = dict(bound.arguments)
            key = CC.signature(name, (), named, invariant=ops.batch_invariant(), storage=ops.storage_dtype())
            if len(self.records[key]) >= KEEP:
                return orig(*args, **kwargs)
            inputs = {k: _clone(v) for k, v in named.items()}
            out = orig(*args, **kwargs)
            written = {k: _clone(named[k]) for k in WRITTEN.get(name, ())}
            self.records[key].append((inputs, _clone(out), written))
            return out
        return wrapper

    def take(self):
        recs, self.records = self.records, defaultdict(list)
        return recs


# --------------------------------------------------------------------------------------------
# replay: one float64 reference per op
# --------------------------------------------------------------------------------------------
def _gemm_family(a):
    if a["conv"] is not None:
        return "conv3x3 nchw" if a["out_nchw"] is not None else "conv3x3"
    if a["geglu"]:
        return "gemm geglu ln-fold" if a["ln"] is not None else "gemm geglu"
    if a["gate_rows"] is not None:
        return "gemm gated"
    if a["ln"] is not None:
        return "gemm ln-fold"
    return "gemm silu/gelu" if a["silu"] or a["gelu"] else "gemm"


def _check_gemm(a, out, invariant, storage):
    """[(family, ratio, note)] of one GEMM launch: its output and, with want_stats, its statistics."""
    res = out[0] if a["want_stats"] else out
    nchw = a["out_nchw"] is not None
    if nchw:
        res = res.permute(0, 2, 3, 1).reshape(-1, res.shape[1])
    ln = None if a["ln"] is None else (a["ln"][1], a["ln"][2])
    y64, bound = CC.gemm64(a["a"], a["w"], a["bias"], residual=a["residual"], gate=a["gate"], rowadd=a["rowadd"],
                           rows_per_batch=a["rows_per_batch"], geglu=a["geglu"], silu=a["silu"], gelu=a["gelu"],
                           conv=a["conv"], gate_rows=a["gate_rows"], ln=ln,
                           out_dtype=torch.float32 if nchw else storage)
    got = res.reshape(y64.shape[0], -1)[:, :y64.shape[1]]
    fam = _gemm_family(a)
    found = [(fam, CC.ratio(got, y64, bound), "")]
    if a["want_stats"]:
        st = out[1]
        fits = CC.slot_check(got, st.t, invariant, storage)
        ok = [bn for bn, r in fits.items() if r <= 1.0]
        kind = ("LNR " if invariant else "") + ("gated" if a["gate_rows"] is not None else "plain")
        # the ratio of the tile width that ran (the best fit); inf when the slot count fits no tile width
        found.append((f"producer stats {kind}", min(fits.values()) if fits else math.inf,
                      f"slots {st.slots} BN {ok[0] if ok else '?'}"))
    return found


def _check(op, a, out, written, invariant, storage):
    """[(family, ratio, note)]; a ratio of -1 marks an exact check that passed, inf one that failed."""
    def exact(family, got, ref):
        return [(family, -1.0 if torch.equal(got, ref) else math.inf, "exact")]
    if op == "gemm":
        return _check_gemm(a, out, invariant, storage)
    if op == "attention":
        kw = {k: a[k] for k in ("batch", "heads", "head_dim", "nq", "n0", "scale", "k1", "v1", "n1", "kv1_batch",
                                "mask")}
        y, b = CC.attention64(a["q"], a["k0"], a["v0"], out_dtype=storage, **kw)
        return [(f"attention d{a['head_dim']}" + (" masked" if a["mask"] is not None else ""), CC.ratio(out, y, b), "")]
    if op == "groupnorm":
        y, b = CC.groupnorm64(a["x"], a["gamma"], a["beta"], batch=a["batch"], hw=a["hw"], groups=a["groups"],
                              eps=a["eps"], silu=a["silu"], out_dtype=storage)
        return [("groupnorm", CC.ratio(out, y, b), "")]
    if op == "layernorm":
        y, b = CC.layernorm64(a["x"], a["gamma"], a["beta"], a["eps"], out_dtype=storage)
        return [("layernorm", CC.ratio(out, y, b), "")]
    if op == "row_stats":
        x = a["x"].reshape(-1, a["x"].shape[-1])
        st = out.t[0].double()
        xd = x.double()
        n = x.shape[1]
        r1 = ((st[:, 0] - xd.sum(1)).abs() / (2 * n * CC.E32 * xd.abs().sum(1) + 1e-30)).max().item()
        r2 = ((st[:, 1] - (xd * xd).sum(1)).abs() / (2 * n * CC.E32 * (xd * xd).sum(1) + 1e-30)).max().item()
        return [("row_stats", max(r1, r2), "")]
    if op == "softmax_rows_":
        y, b = CC.softmax_rows64(a["x"], out_dtype=storage)
        return [("softmax_rows", CC.ratio(out, y, b), "")]
    if op == "scaleu_concat":
        y, b = CC.scaleu64(a["h"], a["skip"], a["b1"], a["s"], batch=a["batch"], height=a["height"],
                           width=a["width"], out_dtype=storage)
        return [("scaleu", CC.ratio(out, y, b), "")]
    if op == "conv_in_select":
        y, b = CC.conv_in_select64(a["x"], a["w0"], a["b0"], a["w1"], a["b1"], a["flags"].cpu(), out_dtype=storage)
        return [("conv_in_select", CC.ratio(out, y, b), "")]
    if op == "timestep_embedding":
        y, b = CC.timestep_embedding64(a["t"], a["dim"], out_dtype=storage)
        return [("timestep_embedding", CC.ratio(out, y, b), "")]
    if op == "fourier_embed":
        y, b = CC.fourier_embed64(a["coords"], a["masks"], a["null_pos"], text=a["text"], null_text=a["null_text"],
                                  mask_mode=a["mask_mode"], dropped=a["dropped"], out_dtype=storage)
        return [("fourier_embed", CC.ratio(out[:, :y.shape[1]], y, b), "")]
    if op == "vae_latent_in":
        y, b = CC.vae_latent_in64(a["z"], a["w"], a["bias"], a["inv_scale"], out_dtype=storage)
        return [("vae_latent_in", CC.ratio(out, y, b), "")]
    if op == "dwconv7x7":
        y, b = CC.dwconv7x7_64(a["x"], a["w49"], a["bias"], a["batch"], a["h"], a["w"], out_dtype=storage)
        return [("dwconv7x7", CC.ratio(out, y, b), "")]
    if op == "segs_inconv":
        y, b, ss, sb = CC.segs_inconv64(a["segs"], a["w"], a["bias"], a["out_size"], out_dtype=storage)
        return [("segs_inconv", max(CC.ratio(out[0], y, b), CC.ratio(out[1], ss, sb)), "")]
    if op == "seg_tokens":
        y = CC.seg_tokens64(a["feat"], a["null_pos"], a["pos"], a["seg_sum"], a["batch"], a["pixels"], a["tokens"])
        return [("seg_tokens", CC.ratio(out, y, 2 * CC.U[storage] * y.abs() + CC.ETA[storage]), "")]
    if op == "im2col_s2":
        return exact("im2col_s2", out, CC.im2col_s2_ref(a["x"], a["batch"], a["h"], a["w"], a["pad01"]))
    if op == "upsample_nearest2x":
        return exact("upsample_nearest2x", out, CC.upsample_nearest2x_ref(a["x"], a["batch"], a["h"], a["w"]))
    if op == "patchify":
        return exact("patchify", out, CC.patchify_ref(a["x"], a["batch"], a["h"], a["w"], a["c"], a["p"]))
    if op == "nchw_f32_to_nhwc_f16":
        return exact("nchw_f32_to_nhwc_f16", out, CC.nchw_to_nhwc_ref(a["x"], a["c_pad"], storage))
    return _check_sampling(op, a, out, written)


def _check_sampling(op, a, out, written):
    """The fp32 sampling updates against the existing float64 references (cases_ddim / cases_dpm / cases_img2img /
    cases_inpaint; PLMS and the latent mean restated in cases_census)."""
    cpu = lambda t: None if t is None else t.detach().double().cpu()  # noqa: E731
    if op == "plms_update":
        olds = [o for o in a["olds"] if o is not None]
        e64, x64 = CC.plms_update64(cpu(a["x"]), cpu(a["e_c"]), cpu(a["e_u"]), a["gs"], [cpu(o) for o in olds],
                                    list(a["coefs"]), a["a_t"], a["a_prev"], a["sqrt_one_minus_at"])
        scale = (1 + abs(a["gs"])) * (1 + sum(abs(c) for c in a["coefs"])) / math.sqrt(a["a_t"])
        mag = scale * sum(cpu(t).abs() for t in [a["x"], a["e_c"]] + ([a["e_u"]] if a["e_u"] is not None else []) + olds)
        r = CC.ratio(written["x_out"].cpu(), x64, E64 * (x64.abs() + mag))
        if written["e_out"] is not None:
            r = max(r, CC.ratio(written["e_out"].cpu(), e64, E64 * (e64.abs() + mag)))
        return [("plms_update", r, "")]
    if op == "latent_mean":
        y = CC.latent_mean64([cpu(x) for x in a["xs"]])
        mag = sum(cpu(x).abs() for x in a["xs"])
        return [("latent_mean", CC.ratio(out.cpu(), y, E64 * (y.abs() + mag)), "")]
    if op == "ddim_update":
        x, e_c, e_u = cpu(a["x"]), cpu(a["e_c"]), cpu(a["e_u"])
        e_out, x_out = torch.empty_like(x), torch.empty_like(x)
        CD.ddim_update(x, e_c, e_u, a["gs"], a["a_t"], a["a_prev"], a["sigma"], a["seed"], a["index"], e_out, x_out)
        z = torch.from_numpy(CN.normals(a["seed"], CN.DDIM_ETA, a["index"], x.numel())).view_as(x)
        scale = (1 + abs(a["gs"])) / math.sqrt(a["a_t"])
        mag = scale * (x.abs() + e_c.abs() + (e_u.abs() if e_u is not None else 0)) + a["sigma"] * z.abs()
        r = CC.ratio(written["x_out"].cpu(), x_out, E64 * (x_out.abs() + mag))
        if written["e_out"] is not None:
            r = max(r, CC.ratio(written["e_out"].cpu(), e_out, E64 * (e_out.abs() + mag)))
        return [("ddim_update", r, "")]
    if op == "dpmpp2m_update":
        x, e_c, e_u, x0p = cpu(a["x"]), cpu(a["e_c"]), cpu(a["e_u"]), cpu(a["x0_prev"])
        x0_out, x_out = torch.empty_like(x), torch.empty_like(x)
        CDP.dpmpp2m_update(x, e_c, e_u, a["gs"], x0p, a["alpha_t"], a["sigma_t"], a["c_x"], a["c_d"], a["w_cur"],
                           a["w_prev"], x0_out, x_out)
        scale = (1 + abs(a["gs"])) * (1 + abs(a["sigma_t"])) / a["alpha_t"] * (1 + abs(a["c_x"]) + abs(a["c_d"])) * (
            1 + abs(a["w_cur"]) + abs(a["w_prev"]))
        mag = scale * (x.abs() + e_c.abs() + (e_u.abs() if e_u is not None else 0) + (x0p.abs() if x0p is not None else 0))
        r = CC.ratio(written["x_out"].cpu(), x_out, E64 * (x_out.abs() + mag))
        if written["x0_out"] is not None:
            r = max(r, CC.ratio(written["x0_out"].cpu(), x0_out, E64 * (x0_out.abs() + mag)))
        return [("dpmpp2m_update", r, "")]
    if op == "noise_latent":
        shape = tuple(out.shape)
        y = CI.x_start64(a["x_init"].reshape((-1,) + shape[1:]), float(a["a"]), a["seed"], shape)
        z = CI.x_start64(a["x_init"].reshape((-1,) + shape[1:]), 0.0, a["seed"], shape)
        mag = a["x_init"].double().cpu().reshape((-1,) + shape[1:]).abs().expand(shape) + z.abs()
        return [("noise_latent", CC.ratio(out.cpu(), y, E64 * (y.abs() + mag)), "")]
    if op == "inpaint_blend":
        ys = CP.inpaint_blend64(a["xs"], a["x0"], a["keep"], a["a"], a["seed"], a["t"])
        shape = tuple(a["xs"][0].shape)
        z = CP.q_value(a["x0"].double().cpu(), 0.0, 1.0, a["seed"], int(a["t"]), shape)
        mag = a["x0"].double().cpu().abs().expand(shape) + z.abs()
        return [("inpaint_blend", max(CC.ratio(o.cpu(), y, E64 * (y.abs() + mag)) for o, y in zip(out, ys)), "")]
    raise AssertionError(f"no reference for {op}")


def replay(recs, worst, what):
    """Check every kept record; fold the worst ratio per op family into `worst`; return failure messages."""
    fails = []
    for key, items in recs.items():
        op, storage, invariant = key[0], getattr(torch, key[1]), key[2]
        for a, out, written in items:
            for family, r, note in _check(op, a, out, written, invariant, storage):
                worst[family] = max(worst.get(family, -1.0), r)
                shapes = {k: tuple(v.shape) for k, v in a.items() if isinstance(v, torch.Tensor)}
                print(f"[census {what}] {family} {note} {shapes} err/bound={r:.3f}")
                if not r <= 1.0:
                    fails.append(f"{what}: {family} {note} {shapes}: err/bound {r:.3g}")
    return fails


# --------------------------------------------------------------------------------------------
# workloads
# --------------------------------------------------------------------------------------------
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
def vae(cuda_device):
    from oracle import torch_oracle as TO
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.weights import synth_tensor
    with torch.device("meta"):
        m = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    m = m.to_empty(device=cuda_device).eval()
    m.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), cases.WEIGHT_SEED) for k, v in m.state_dict().items()},
                      strict=True)
    return m


def _att_masks(gi):
    from instancediffusion_b200 import ops
    counts = gi["masks"].sum(-1).round().int().contiguous()
    return ops.boxes_to_attmask(gi["boxes"].float().contiguous(), counts)


def _workload_mixed64(unet, dev):
    from instancediffusion_b200 import synthetic
    gti = unet.grounding_tokenizer_input
    inputs, scales, restored = [], [], []
    for k, seed in enumerate(range(301, 306)):
        ia, uca = synthetic.make_sampler_inputs(gti, 1, 2, seed, "box", device=dev)
        if k == 1:
            ia["grounding_input"]["att_masks"] = _att_masks(ia["grounding_input"])
        t = torch.full((1,), 100 + 150 * k, dtype=torch.long, device=dev)
        inputs += [dict(x=ia["x"], timesteps=t, context=ia["context"], grounding_input=ia["grounding_input"]),
                   dict(x=ia["x"] * 0.7, timesteps=t, context=uca)]
        scales += [(1.0, 0.0, 0.36, 1.0, 0.0)[k]] * 2
        restored += [k == 3] * 2
    unet.forward_batched(inputs, scales=scales, restored=restored)


def _workload_case(unet, dev, name):
    import test_parity_r2_gpu as P
    spec = cases.UNET_EXTRA_CASES[name]
    P._set_flavor(unet.position_net, spec["flavor"])
    unet.clear_caches()
    try:
        inp, uc, ts = P._inputs(unet, spec, dev)
        cond = dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=inp["grounding_input"])
        if spec.get("uncond"):
            unet.forward_batched([cond, dict(x=inp["x"], timesteps=ts, context=uc)])
        else:
            unet(cond)
    finally:
        P._set_flavor(unet.position_net, "box")
        unet.clear_caches()


def _workload_decode(vae, dev):
    g = torch.Generator().manual_seed(7)
    vae.decode((torch.randn((1, 4, 64, 64), generator=g) * 0.9).to(dev))


def _workload_modules(vae, dev):
    """The two entry points the UNet and the decode above never call: row_stats (a gated self-attention block run as
    a module) and nchw_f32_to_nhwc_f16 (the first-stage encoder's input)."""
    from instancediffusion_b200.ldm.modules.attention import GatedSelfAttentionDense
    cases.run_module_case("gated_sa_L0", cases.MODULE_CASES["gated_sa_L0"], GatedSelfAttentionDense, device=dev)
    g = torch.Generator().manual_seed(43)
    vae.encoder((torch.randn((1, 3, 64, 64), generator=g) * 0.5).to(dev))


WORKLOADS = {
    "forward_batched 64x64 mixed": lambda unet, vae, dev: _workload_mixed64(unet, dev),
    "96x96 latent": lambda unet, vae, dev: _workload_case(unet, dev, "lat96"),
    "batch 4+4, 8 instances": lambda unet, vae, dev: _workload_case(unet, dev, "b4n8"),
    "mask flavour": lambda unet, vae, dev: _workload_case(unet, dev, "mask"),
    "VAE decode 64x64 -> 512^2": lambda unet, vae, dev: _workload_decode(vae, dev),
    "module forwards": lambda unet, vae, dev: _workload_modules(vae, dev),
}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_launch_census(cuda_device, unet, vae, monkeypatch, dtype, mode):
    """Every workload's distinct launches against float64; every wrapped op seen; in batch-invariant mode at least
    one stored-statistics (LNR) producer of each epilogue mode, and a per-image gated launch with a zero gate."""
    from instancediffusion_b200 import ops
    from instancediffusion_b200.utils.model import set_alpha_scale
    t0 = time.time()
    rec = Recorder(monkeypatch, FORWARD_OPS)
    seen, worst, fails, lnr = set(), {}, [], set()
    unet.use_cuda_graph = False
    try:
        with ops.storage(DTYPES[dtype]):
            ops.set_batch_invariant(MODES[mode])
            for wname, run in WORKLOADS.items():
                with torch.no_grad():
                    run(unet, vae, cuda_device)
                torch.cuda.synchronize()
                recs = rec.take()
                print(f"[census] {wname} {mode} {dtype}: {len(recs)} distinct signatures")
                for key, items in recs.items():
                    seen.add(key[0])
                    if key[0] == "gemm" and key[2]:
                        a = items[0][0]
                        if a["want_stats"]:
                            lnr.add("gated" if a["gate_rows"] is not None else "plain")
                        if a["gate_rows"] is not None and any(bool((it[0]["gate_rows"] == 0).any()) for it in items):
                            lnr.add("zero gate")
                fails += replay(recs, worst, f"{wname} {mode} {dtype}")
                del recs
    finally:
        ops.set_batch_invariant(False)
        unet.use_cuda_graph = True
        set_alpha_scale(unet, 1)
        unet.undo_first_conv_restore()
        unet.clear_caches()
    for fam in sorted(worst):
        print(f"[census {mode} {dtype}] worst err/bound {fam}: {worst[fam]:.3f}" + (" (exact)" if worst[fam] < 0 else ""))
    print(f"[census {mode} {dtype}] wall time {time.time() - t0:.1f} s")
    missing = set(FORWARD_OPS) - seen
    assert not missing, f"ops never launched: {sorted(missing)}"
    if MODES[mode]:
        assert {"plain", "gated", "zero gate"} <= lnr, f"invariant census lacks LNR launches: has {sorted(lnr)}"
    assert not fails, "\n".join(fails[:40])


def test_sampling_kernel_census(cuda_device, unet, monkeypatch):
    """One short sample_requests run per mode, four requests (PLMS Multi-instance, DDIM eta 0.5, DPM-Solver++, an
    inpainting x_init request): every sampling-update launch against float64."""
    from functools import partial
    from instancediffusion_b200 import ops, synthetic
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, sample_requests
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(cuda_device)
    gti = unet.grounding_tokenizer_input
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    S = 4
    common = dict(guidance_scale=7.5, alpha_generator_func=agen, S=S, shape=(1, 4, 64, 64))
    mis_in, mis_uc = synthetic.make_sampler_inputs(gti, 1, 2, 801, "box", mis=True, device=cuda_device)
    ins = [synthetic.make_sampler_inputs(gti, 1, 2, 802 + i, "box", device=cuda_device) for i in range(3)]
    x_init = torch.randn((1, 4, 64, 64), generator=torch.Generator().manual_seed(9)).to(cuda_device)
    worst, fails = {}, []
    for mode, inv in MODES.items():
        reqs = [Request(input=mis_in, uc=mis_uc, mis=0.36, **common),
                Request(input=ins[0][0], uc=ins[0][1], sampler="ddim", eta=0.5, seed=31, **common),
                Request(input=ins[1][0], uc=ins[1][1], sampler="dpmpp_2m", **common),
                Request(input=ins[2][0], uc=ins[2][1], x_init=x_init, strength=0.8,
                        repaint_mask=CP.box_mask(1, 512, (96, 352, 128, 416)), seed=32, **common)]
        rec = Recorder(monkeypatch, SAMPLING_OPS)
        ops.set_batch_invariant(inv)
        try:
            sample_requests(unet, diffusion, reqs, S)
            torch.cuda.synchronize()
        finally:
            ops.set_batch_invariant(False)
            set_alpha_scale(unet, 1)
            unet.undo_first_conv_restore()
            monkeypatch.undo()
        recs = rec.take()
        print(f"[census] sample_requests {mode}: {len(recs)} distinct signatures")
        assert {k[0] for k in recs} == set(SAMPLING_OPS), sorted({k[0] for k in recs})
        fails += replay(recs, worst, f"sample_requests {mode}")
    for fam in sorted(worst):
        print(f"[census sampling] worst err/bound {fam}: {worst[fam]:.3f}")
    assert not fails, "\n".join(fails[:40])
