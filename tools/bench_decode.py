#!/usr/bin/env python
"""Cost of turning finished requests into images: eight one-image config-2-shaped requests (512x512 / latent 64x64,
8 box instances, CFG 7.5, PLMS, fp16, seeded synthetic weights and inputs) that finish in one tick, two ways on the same
card, passes alternated:

  batched    what `SamplingEngine` / `sample_requests` do for `output="image"`: the eight latents decoded together
             (`batched.decode_latents`, at most `max_decode_batch` = 8 images per decoder forward), the decode_to_image
             kernel, and the uint8 images copied to the host;
  one_by_one the reference's inference.py:96-125 per request: `decode` at batch 1, torch.clamp(x, -1, 1) * 0.5 + 0.5,
             the fp32 image copied to the host, * 255 and astype(np.uint8) in numpy.

The latents come from one `SamplingEngine` run of the eight requests with `output="latent"` (--steps, default 10: the
decode does not depend on the step count).  Reports per arm the milliseconds per image (host clock around the whole
arm, ending with the images on the host; median, min and max over --reps), the bytes copied to the host (counted from
the shapes), and the byte difference between the arms; for the epilogue kernel alone, its time over --kernel-iters
launches on the (8, 3, 512, 512) decoder output in fp32 and in the 16-bit storage type (CUDA events) against its
bandwidth bound (4- or 2-byte reads plus 1-byte writes per element at 3.35 TB/s, the H100 SXM data sheet's HBM3 rate);
and the card's name and power limit.

  python tools/bench_decode.py [--reps 5] [--steps 10] [--out results/decode.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from functools import partial

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_REQ, N_INST, GUIDANCE = 8, 8, 7.5
HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decode.py: no CUDA device (there is no CPU path)")

    from bench import ClockSampler
    from bench_requests import gpu_info
    from oracle import torch_oracle as TO
    from instancediffusion_b200 import ops, synthetic
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.ldm.models.diffusion.batched import Request, decode_latents
    from instancediffusion_b200.ldm.models.diffusion.engine import SamplingEngine
    from instancediffusion_b200.ldm.models.diffusion.ldm import LatentDiffusion
    from instancediffusion_b200.utils.model import alpha_generator
    from instancediffusion_b200.weights import build_unet, synth_tensor

    device = torch.device("cuda:0")
    model = build_unet("box", device, seed=0)
    sd_conv = torch.load(os.path.join(ROOT, "tests", "golden", "sd15_first_conv.pt"), map_location="cpu")
    model.restore_first_conv_from_SD = lambda: (None if getattr(model, "_first_conv_restored", False)
                                                else model.set_sd_first_conv(sd_conv))
    model.restore_first_conv_from_SD()  # the engine's per-image conv needs the SD1.5 conv weights known
    model.undo_first_conv_restore()
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)
    with torch.device("meta"):
        vae = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    vae = vae.to_empty(device=device).eval()
    vae.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), 0) for k, v in vae.state_dict().items()},
                        strict=True)

    agen = partial(alpha_generator, type=[0.8, 0.0, 0.2])
    eng = SamplingEngine(model, diffusion, max_batch=2 * N_REQ)
    tickets = []
    for k in range(N_REQ):
        inp, uc = synthetic.make_sampler_inputs(model.grounding_tokenizer_input, 1, N_INST, 900 + k, "box",
                                                device=device)
        tickets.append(eng.submit(Request(input=inp, uc=uc, guidance_scale=GUIDANCE, alpha_generator_func=agen,
                                          shape=(1, 4, 64, 64), S=args.steps)))
    done, ticks = {}, 0
    while eng.queued or eng.live:
        out = eng.step()
        ticks += 1
        if out:
            assert len(out) == N_REQ, f"{len(out)} of {N_REQ} requests finished in tick {ticks}"
        done.update(out)
    latents = [done[t].float().contiguous() for t in tickets]

    def batched():
        imgs = decode_latents(vae, latents, 8)
        return [im.cpu().numpy() for im in imgs]

    def one_by_one():
        imgs = []
        for z in latents:
            sample = vae.decode(z)[0]
            sample = torch.clamp(sample, min=-1, max=1) * 0.5 + 0.5
            sample = sample.cpu().numpy().transpose(1, 2, 0) * 255
            imgs.append(sample.astype(np.uint8))
        return imgs

    arms = {"batched": batched, "one_by_one": one_by_one}
    outs = {name: fn() for name, fn in arms.items()}  # warm-up
    torch.cuda.synchronize()
    runs = {name: [] for name in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            with ClockSampler(0) as clk:
                t0 = time.perf_counter()
                outs[name] = fn()
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
            runs[name].append({"ms_per_image": 1e3 * t / N_REQ, "clocks": clk.summary()})
    a = np.stack([o.reshape(512, 512, 3) for o in outs["batched"]]).astype(np.int32)
    b = np.stack([o.reshape(512, 512, 3) for o in outs["one_by_one"]]).astype(np.int32)
    host_bytes = {"batched": N_REQ * 512 * 512 * 3, "one_by_one": N_REQ * 3 * 512 * 512 * 4}
    summary = {}
    for name, rs in runs.items():
        ms = sorted(r["ms_per_image"] for r in rs)
        summary[name] = {"decode_ms_per_image_median": ms[len(ms) // 2], "min": ms[0], "max": ms[-1],
                         "bytes_to_host": host_bytes[name]}
    summary["speedup_one_by_one_over_batched"] = (summary["one_by_one"]["decode_ms_per_image_median"]
                                                  / summary["batched"]["decode_ms_per_image_median"])

    # the epilogue kernel alone on the decoder output of the eight images
    x32 = vae.decode(torch.cat(latents))
    kernel = {}
    for name, x in (("fp32_in", x32), ("storage_in", x32.to(ops.storage_dtype()))):
        img = torch.empty((N_REQ, 512, 512, 3), dtype=torch.uint8, device=device)
        for _ in range(10):
            ops.decode_to_image(x, img)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.kernel_iters):
            ops.decode_to_image(x, img)
        ev[1].record()
        torch.cuda.synchronize()
        us = ev[0].elapsed_time(ev[1]) * 1e3 / args.kernel_iters
        nbytes = x.numel() * (x.element_size() + 1)
        bound_us = nbytes / HBM_BYTES_PER_S * 1e6
        kernel[name] = {"us": us, "bytes": nbytes, "bound_us_at_3.35TB/s": bound_us, "share_of_bound": bound_us / us,
                        "achieved_TB/s": nbytes / us * 1e-6}
    line = {
        "workload": f"{N_REQ} one-image config2-shaped requests (512x512, {N_INST} box instances, CFG {GUIDANCE}, "
                    f"{args.steps}-step PLMS, fp16) finishing in one tick (tick {ticks}); decode of their latents",
        "gpu": gpu_info(), "reps": args.reps, "summary": summary, "epilogue_kernel": kernel, "runs": runs,
        "bytes_batched_vs_one_by_one": {"max_abs_diff": int(np.abs(a - b).max()),
                                        "fraction_differing": float((a != b).mean())},
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
