#!/usr/bin/env python
"""Cost of starting image-to-image requests from images: eight one-image 512x512 requests (seeded synthetic SD1.5-shaped
VAE weights, random uint8 images on the device), their latents made two ways on the same card, passes alternated:

  batched    what `sample_requests` / `SamplingEngine` do for `init_image` requests: the eight images encoded together
             (`batched.encode_images`, at most `max_encode_batch` = 8 images per encoder forward: the image-in conv
             kernel, the encoder, the fused posterior kernel with each request's seed);
  one_by_one the path before `init_image`: per request, torch's u / 127.5 - 1 and NCHW permute, then
             `AutoencoderKL.encode` at batch 1 (padded copy + conv GEMM input conv, torch quant_conv and posterior with
             the global CPU generator's noise).

Reports per arm the milliseconds per image until the latents are on the device (host clock around the arm, ending in
a device synchronise; median, min and max over --reps).  Kernel timings (CUDA events around each launch, L2 flushed
before it by writing a 256 MB buffer, median of --kernel-iters launches):
  * the image-in kernel against what it replaces, the 64-channel padded NHWC copy of the normalised fp32 image plus
    the conv GEMM, at batch 1 and 8 (512x512, 3 -> 128 channels); useful FLOPs 2 * 27 * 128 per pixel;
  * the posterior kernel on the (8, 8, 64, 64) conv_out, against its bandwidth bound (fp32 reads of 8 planes and
    writes of 4 at 3.35 TB/s, the H100 SXM data sheet's HBM3 rate).
And the card's name and power limit.

  python tools/bench_encode.py [--reps 5] [--kernel-iters 21] [--out results/encode.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_REQ, SIZE = 8, 512
HBM_BYTES_PER_S = 3.35e12


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def time_launches(fn, iters: int, flush: torch.Tensor):
    """Median, min and max microseconds of `fn` over `iters` launches, each after an L2 flush (CUDA events)."""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]) * 1e3)
    return {"us_median": _median(ts), "us_min": min(ts), "us_max": max(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=21)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode.py: no CUDA device (there is no CPU path)")

    from bench_requests import gpu_info
    from oracle import torch_oracle as TO
    from instancediffusion_b200 import ops
    from instancediffusion_b200.ldm.models.autoencoder import AutoencoderKL
    from instancediffusion_b200.ldm.models.diffusion.batched import encode_images
    from instancediffusion_b200.weights import synth_tensor

    device = torch.device("cuda:0")
    with torch.device("meta"):
        vae = AutoencoderKL(dict(TO.VAE_DDCONFIG), 4, TO.VAE_SCALE)
    vae = vae.to_empty(device=device).eval()
    vae.load_state_dict({k: synth_tensor("vae." + k, tuple(v.shape), 0) for k, v in vae.state_dict().items()},
                        strict=True)
    g = torch.Generator().manual_seed(5)
    images = [torch.randint(0, 256, (1, SIZE, SIZE, 3), generator=g, dtype=torch.uint8).to(device)
              for _ in range(N_REQ)]
    seeds = [1000 + k for k in range(N_REQ)]

    def batched():
        return encode_images(vae, images, seeds, 8)

    def one_by_one():
        out = []
        for im in images:
            x = (im.float() / 127.5 - 1).permute(0, 3, 1, 2).contiguous()
            out.append(vae.encode(x))
        return out

    arms = {"batched": batched, "one_by_one": one_by_one}
    with torch.no_grad():
        for fn in arms.values():
            fn()  # warm-up
        torch.cuda.synchronize()
        runs = {name: [] for name in arms}
        for _ in range(args.reps):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                runs[name].append(1e3 * (time.perf_counter() - t0) / N_REQ)
    summary = {}
    for name, ms in runs.items():
        ms = sorted(ms)
        summary[name] = {"encode_ms_per_image_median": _median(ms), "min": ms[0], "max": ms[-1]}
    summary["speedup_one_by_one_over_batched"] = (summary["one_by_one"]["encode_ms_per_image_median"]
                                                  / summary["batched"]["encode_ms_per_image_median"])

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    p = vae.encoder.pk()
    kernels = {}
    for B in (1, 8):
        img = torch.cat(images[:B]) if B > 1 else images[0]
        x = (img.float() / 127.5 - 1).permute(0, 3, 1, 2).contiguous()
        tok = torch.empty((B * SIZE * SIZE, 128), dtype=ops.storage_dtype(), device=device)
        pad = torch.empty((B * SIZE * SIZE, 64), dtype=ops.storage_dtype(), device=device)
        new = time_launches(lambda: ops.encode_image_in(img, p["w_img"], p["b_in"], out=tok), args.kernel_iters, flush)
        copy = time_launches(lambda: ops.nchw_f32_to_nhwc_f16(x, 64, out=pad), args.kernel_iters, flush)
        gemm = time_launches(lambda: ops.gemm(pad, p["w_in"], p["b_in"], conv=(B, SIZE, SIZE, 64)), args.kernel_iters,
                             flush)
        both = time_launches(lambda: ops.gemm(ops.nchw_f32_to_nhwc_f16(x, 64, out=pad), p["w_in"], p["b_in"],
                                              conv=(B, SIZE, SIZE, 64)), args.kernel_iters, flush)
        useful = 2.0 * 27 * 128 * B * SIZE * SIZE
        kernels[f"image_in_b{B}"] = {
            "image_in_kernel": new, "pad64_copy": copy, "conv_gemm_k576": gemm, "pad64_copy_plus_gemm": both,
            "useful_GFLOP": useful * 1e-9, "image_in_useful_TFLOP/s": useful / new["us_median"] * 1e-6,
            "speedup_padded_over_image_in": both["us_median"] / new["us_median"]}
    hb = vae.encoder._encode_tokens(ops.encode_image_in(torch.cat(images), p["w_img"], p["b_in"]), N_REQ, SIZE, SIZE)
    pa = vae.pk()
    sarr, idx = ops.seed_array(seeds, device), torch.zeros((N_REQ,), dtype=torch.int32, device=device)
    zout = torch.empty((N_REQ, 4, SIZE // 8, SIZE // 8), dtype=torch.float32, device=device)
    post = time_launches(lambda: ops.encode_posterior(hb, pa["wq"], pa["bq"], 0.18215, sarr, idx, out=zout),
                         args.kernel_iters, flush)
    nbytes = 4.0 * (hb.numel() + zout.numel())
    bound_us = nbytes / HBM_BYTES_PER_S * 1e6
    kernels["posterior_b8_64x64"] = dict(post, bytes=nbytes, **{"bound_us_at_3.35TB/s": bound_us,
                                                                 "share_of_bound": bound_us / post["us_median"]})
    line = {
        "workload": f"{N_REQ} one-image {SIZE}x{SIZE} image-to-image requests: uint8 images on the device to latents "
                    f"on the device (SD1.5 VAE shapes, seeded synthetic weights, {ops.storage_dtype()} storage)",
        "gpu": gpu_info(), "reps": args.reps, "summary": summary, "kernels": kernels, "runs_ms_per_image": runs,
    }
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
