#!/usr/bin/env python
"""Cost of inpainting requests (`Request.repaint_mask`), three measurements on seeded synthetic weights and inputs:

1. The blend kernel (`ops.inpaint_blend`, one launch per request and step) against the drop-in samplers' torch blend
   (`diffusion.q_sample` + `mask * q + (1 - mask) * x` per trajectory, SamplingRun.begin's `blend`), at batch 1, 4 and
   8 of a 64x64 latent with one trajectory and at batch 4 with the 9 trajectories of an 8-instance Multi-instance
   request; the mask repaints a 256x288-pixel box.  CUDA events around each call after an L2 flush (256 MB write),
   median, min and max of --kernel-iters calls, next to the time the kernel's bytes take at 3.35 TB/s (the H100 SXM
   data sheet's HBM3 rate).
2. End to end: two config-2-shaped requests (batch 4, 512x512 / latent 64x64, 8 box instances, CFG 7.5, alpha schedule
   [0.8, 0, 0.2], 50-step PLMS, fp16) from x_init at strength 1 through `sample_requests`, with the box repaint mask
   and without it, alternated over --reps timed passes (CUDA events; median, min, max).
3. The paste-back (`batched.paste_back`, one `torch.where` over the image) per 512x512 image next to the batch-4 decode
   (`decode_latents` of the seeded first stage), CUDA events, median of --kernel-iters.
And the card's name, power limit and max SM clock, read in the same run.

  python tools/bench_inpaint.py [--reps 3] [--kernel-iters 21] [--steps 50] [--out results/inpaint.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from dataclasses import replace
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

BATCH, N_INST, GUIDANCE = 4, 8, 7.5
BOX = (128, 384, 96, 384)  # repainted pixels (y0, y1, x0, x1) of the 512x512 image
HBM_BYTES_PER_S = 3.35e12


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def _box_mask(b, device):
    m = torch.zeros((b, 512, 512), dtype=torch.bool, device=device)
    m[:, BOX[0]:BOX[1], BOX[2]:BOX[3]] = True
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=21)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint.py: no CUDA device (there is no CPU path)")

    from bench_encode import time_launches
    from bench_requests import gpu_info
    from oracle import torch_oracle as TO
    import cases
    from instancediffusion_b200 import ops, synthetic
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.ldm.models.diffusion.batched import (Request, decode_latents, keep_mask, paste_back,
                                                                      sample_requests)
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale
    from instancediffusion_b200.weights import build_unet, synth_tensor

    device = torch.device("cuda:0")
    gpu = gpu_info()
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    g = torch.Generator().manual_seed(0)

    # 1. the blend kernel against the torch blend
    t = 801
    a = (float(diffusion.sqrt_alphas_cumprod[t]), float(diffusion.sqrt_one_minus_alphas_cumprod[t]))
    kernels = {}
    for B, count in ((1, 1), (4, 1), (8, 1), (4, 9)):
        xs = [torch.randn((B, 4, 64, 64), generator=g).to(device) for _ in range(count)]
        outs = [torch.empty_like(x) for x in xs]
        x0 = torch.randn((1, 4, 64, 64), generator=g).to(device)
        keep = keep_mask(_box_mask(1, device))
        mask = keep.float()[:, None]
        ts = torch.full((B,), t, dtype=torch.long, device=device)
        x0b = x0.expand(B, 4, 64, 64).contiguous()

        def torch_blend():
            q = diffusion.q_sample(x0b, ts)
            return [q * mask + (1. - mask) * x for x in xs]
        fused = time_launches(lambda: ops.inpaint_blend(xs, outs, x0, keep, a, 7, t), args.kernel_iters, flush)
        ref = time_launches(torch_blend, args.kernel_iters, flush)
        n = xs[0].numel()
        kept = keep.float().mean().item()
        nbytes = 4 * count * n + 4 * count * n * (1 - kept) + 4 * n * kept + keep.numel()  # outs, repainted x, x0, keep
        kernels[f"b{B}_x{count}"] = {"inpaint_blend": fused, "torch_blend": ref,
                                     "speedup_median": ref["us_median"] / fused["us_median"],
                                     "bytes": nbytes, "kept_fraction": kept,
                                     "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6}

    # 2. end to end through sample_requests
    model = build_unet("box", device, seed=0)
    sd_conv = torch.load(os.path.join(ROOT, "tests", "golden", "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(sd_conv))
    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    shape = (BATCH, 4, 64, 64)
    reqs = []
    for k in range(2):
        inp, uc = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, BATCH, N_INST, 900 + k, "box",
                                                device=device)
        reqs.append(Request(input=inp, uc=uc, guidance_scale=GUIDANCE, alpha_generator_func=agen, shape=shape,
                            x_init=torch.randn(shape, generator=g).to(device), seed=100 + k,
                            repaint_mask=_box_mask(1, device)))

    def run(masked):
        model.undo_first_conv_restore()
        set_alpha_scale(model, 1)
        rs = [replace(r, input=dict(r.input), repaint_mask=r.repaint_mask if masked else None) for r in reqs]
        return sample_requests(model, diffusion, rs, args.steps, max_batch=4 * BATCH)

    arms = {"repaint_mask": True, "no_mask": False}
    for masked in arms.values():  # warm-up: graph capture, hoisted tensors
        run(masked)
    torch.cuda.synchronize()
    e2e = {name: [] for name in arms}
    for _ in range(args.reps):
        for name, masked in arms.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            torch.cuda.synchronize()
            ev[0].record()
            run(masked)
            ev[1].record()
            torch.cuda.synchronize()
            e2e[name].append(ev[0].elapsed_time(ev[1]) * 1e-3)
    end_to_end = {name: {"seconds_median": _median(v), "seconds_min": min(v), "seconds_max": max(v), "runs": v,
                         "images_per_s_median": 2 * BATCH / _median(v)} for name, v in e2e.items()}
    end_to_end["overhead_median"] = (end_to_end["repaint_mask"]["seconds_median"]
                                     / end_to_end["no_mask"]["seconds_median"] - 1)
    del model

    # 3. the paste-back next to the decode
    with torch.device("meta"):
        vae = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    vae = vae.to_empty(device=device).eval()
    vae.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), cases.WEIGHT_SEED)
                         for k, v in vae.state_dict().items()}, strict=True)
    z = torch.randn((BATCH, 4, 64, 64), generator=g).to(device)
    src = torch.randint(0, 256, (1, 512, 512, 3), generator=g, dtype=torch.uint8).to(device)
    req = Request(input={}, init_image=src, repaint_mask=_box_mask(1, device))
    with torch.no_grad():
        img = decode_latents(vae, [z], BATCH)[0]
        dec = time_launches(lambda: decode_latents(vae, [z], BATCH), args.kernel_iters, flush)
    paste = time_launches(lambda: paste_back(req, img), args.kernel_iters, flush)
    paste_cost = {"decode_batch4": dec, "paste_back_batch4": paste,
                  "decode_us_per_image": dec["us_median"] / BATCH, "paste_back_us_per_image": paste["us_median"] / BATCH}

    line = {
        "gpu": gpu, "storage": str(ops.storage_dtype()),
        "blend_kernel": kernels,
        "end_to_end": dict(end_to_end, workload=f"2 requests of batch {BATCH} 512x512, {N_INST} box instances, "
                                                f"{args.steps}-step PLMS, CFG {GUIDANCE}, alpha [0.8, 0, 0.2], "
                                                f"x_init at strength 1, repaint box {BOX}", reps=args.reps),
        "paste_back": paste_cost,
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
