"""Many independent sampling requests advanced in lock step (not a reference module).

A deployment that gets one layout per user would otherwise run one `sample()` call per request: every forward
then has the batch of that one request (cond + uncond of one image: 512 GEMM rows at the 16x16 level against
128-row tiles).  `sample_requests` evaluates, at every step, the live trajectories of all requests together in
`forward_batched` chunks of up to `max_batch` images, each image with its own request's fuser scale (alpha
schedule) and first-conv state.  Per request the arithmetic is that of its own sampler: each request is a
`SamplingRun` (_plms_common.py), the run its sampler's `sample()` drives, on the sampler kind `SAMPLERS[sampler]`
(`PLMSBase`, `DDIMBase`, `DPMSolverBase`) with its own guidance scale, seed and Multi-instance merge at its own step
int(steps * mis), where steps is the length of the schedule (`schedule_steps`: S + 1 for some S, e.g. 31 for S = 30).
A DDIM request's eta noise is keyed by its own seed and the step, so it does not depend on the other requests.  An
image-to-image request (`x_init`, `strength`) starts at its sampler's step k0 from x_init noised there; in lock step it
joins the others at step k0, so every request ends with the last step.  `_RequestState` adds to the run what the
request drivers need: what the model was at admission and the batched evaluation with per-image fuser scales and
convs.  `SamplingEngine` (engine.py) drives it too: `sample_requests` is the lock-step driver on top of it.  A request
with `output="image"` gets the image of its latent instead: the drivers decode the latents of the image requests that finish
together in batched first-stage forwards (`decode_latents`), eagerly and apart from the UNet's caches and graphs.  A
request may also start from an image (`init_image`, uint8): the drivers encode the images of the requests that start
together in batched first-stage forwards (`encode_images`), eagerly, before those requests' start latents, and the
request then runs as if it had been given x_init = autoencoder.encode_images(init_image, seed=its seed).  An
image-to-image request may also repaint part of its image (`repaint_mask`, inpainting): before every evaluation the
latent cells outside the mask are replaced by x_init noised to the step's timestep, with a noise keyed by the request's
seed and the timestep (`SamplingRun.inpaint`), so everything outside the mask stays the source's; an image output of
an `init_image` request takes the source's pixels outside the mask (`paste_back`).

Contract: each returned latent equals, within floating-point tolerance, what `PLMSSampler.sample()` (input dict,
mis = 0), `PLMSSamplerInst.sample()` (input list [global, instance_1 .. instance_n]), `DDIMSampler.sample(eta=,
seed=)` or `DPMSolverSampler.sample()` returns for that request alone on the model in the state it had when
`sample_requests` was called; for an `init_image` request, what the same request with x_init =
`AutoencoderKL.encode_images(init_image, seed=seed)` returns (bit for bit in batch-invariant mode); for an inpainting
request (`repaint_mask`), what its sampler's `sample_loop(mask=keep, x0=x_init, x_init=x_init, ...)` returns alone
with `diffusion.q_sample` drawing its noise from the seeded blend stream (`ops.inpaint_blend`) instead of torch's
global generator.  Afterwards the model's fuser scale and first-conv swap are what a sequential run of the same
requests would leave.
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import torch

from ...modules.attention import GatedSelfAttentionDense
from ...modules.diffusionmodules.util import make_ddim_timesteps
from ._plms_common import PLMSBase, RequestPlan, SamplingRun, check_init, plan_chunks, resolve_seed
from .ddim import DDIMBase
from .dpm_solver import DPMSolverBase


@dataclass
class Request:
    """One sampling request.  `input`: the dict `PLMSSampler.sample` takes, or the list [global, inst_1 .. inst_n]
    of `PLMSSamplerInst.sample`; `shape`: (B, 4, H, W) of its latent (may be omitted when input x is given);
    `mis`: the Multi-instance fraction (list inputs only).  `S`: the request's step count; `sample_requests` takes it
    from the call (S, if given, must equal it), `SamplingEngine` requires it.  `mask` / `x0` (the reference's inpainting,
    whose noise comes from torch's global generator and so depends on what ran before) are not supported and raise:
    inpainting requests use `repaint_mask`.  `sampler`: a name of `SAMPLERS`: "plms", "ddim" (`DDIMSampler.sample`: input dict only)
    with its `eta` and `seed` (None at eta > 0: one draw from torch's default CPU generator when `sample_requests`
    starts or at `submit`, in request order), or "dpmpp_2m" (`DPMSolverSampler.sample`: input dict only, eta = 0).  `x_init`: a latent of
    shape (1 or B, C, H, W) to start image-to-image sampling from, which runs the last int(N * strength) of the N schedule steps (the samplers' `x_init` / `strength`); the start noise is
    keyed by `seed`, drawn as for DDIM when None.  `output`: "latent" (the sampler's latent) or "image" (that latent
    decoded by the driver's `autoencoder` to uint8 (B, 8H, 8W, 3) on the device, `AutoencoderKL.decode_images`).
    `init_image`: instead of x_init, uint8 RGB images (1 or B, 8H, 8W, 3) on any device, which the driver's
    `autoencoder` encodes with the request's seed (`AutoencoderKL.encode_images(init_image, seed=seed)`) into the x_init
    the request starts from; one image on a B > 1 request is encoded once and broadcast.  The request is not modified:
    the latent stays with the driver.

    `repaint_mask`: inpainting, a bool or uint8 tensor (1 or B, 8H, 8W) at pixel resolution on any device, nonzero =
    regenerate this pixel; it needs x_init or init_image, the source of the kept region.  A latent cell (y, x) is
    repainted if any pixel of [8y, 8y+8) x [8x, 8x+8) is; before every evaluation (not the corrector's of a first PLMS
    step) every other cell of every trajectory is set to q_sample(x_init, t) at the step's timestep t, its noise keyed
    by (seed, t), as `PLMSBase.sample_loop(mask=, x0=x_init)` blends (plms.py:99-103).  `strength` keeps its meaning:
    1 is classic inpainting from x_init noised at the first timestep, below 1 the masked region is also repainted
    SDEdit-style from the noised source.  Every sampler kind takes it, and Multi-instance requests blend every
    trajectory before the merge with the same source latent (as `sample_loop(mis=, mask=, x0=)`; the drop-in
    `PLMSSamplerInst.sample` ignores mask / x0, as the reference's does).  An `output="image"` request started from
    `init_image` returns the source's bytes wherever the mask is zero (`paste_back`); one started from x_init has no
    source pixels and returns the decoded image as it is."""
    input: Union[dict, List[dict]]
    uc: Optional[torch.Tensor] = None
    guidance_scale: float = 1.0
    alpha_generator_func: Optional[Callable[[int], List[float]]] = None
    mis: float = 0.0
    shape: Optional[Tuple[int, ...]] = None
    S: Optional[int] = None
    mask: Optional[torch.Tensor] = None
    x0: Optional[torch.Tensor] = None
    sampler: str = "plms"
    eta: float = 0.0
    seed: Optional[int] = None
    x_init: Optional[torch.Tensor] = None
    strength: float = 1.0
    output: str = "latent"
    init_image: Optional[torch.Tensor] = None
    repaint_mask: Optional[torch.Tensor] = None


SAMPLERS = {kind.sampler: kind for kind in (PLMSBase, DDIMBase, DPMSolverBase)}
OUTPUTS = ("latent", "image")


def plan_step(plans: Sequence[RequestPlan], step: int, max_batch: int) -> List[List[Tuple[int, int]]]:
    """Forward chunks of one evaluation at `step`: every live trajectory of every request."""
    slots = [(r, k) for r, p in enumerate(plans) for k in range(p.live(step))]
    return plan_chunks(slots, plans, max_batch)


def _inputs_of(req: Request) -> List[dict]:
    return req.input if isinstance(req.input, (list, tuple)) else [req.input]


def schedule_steps(S: int, ddpm_timesteps: int = 1000) -> int:
    """Steps of the PLMS schedule the samplers build for S (PLMSBase.make_schedule, 'uniform'): the timesteps
    range(0, ddpm_timesteps, ddpm_timesteps // S), which is more than S when S does not divide ddpm_timesteps."""
    return len(make_ddim_timesteps("uniform", int(S), int(ddpm_timesteps)))


def check_requests(requests: Sequence[Request], S: int, max_batch: int, ddpm_timesteps: int = 1000) -> List[RequestPlan]:
    """Validate the requests of one `sample_requests` call and describe them for the planner.  All must share the
    step count S, the latent height x width and the context length; mask / x0 inpainting is not supported (inpainting
    requests give `repaint_mask`).
    A Multi-instance request merges before step int(schedule_steps(S) * mis), as PLMSSamplerInst does (an
    image-to-image one only if that step lies after its start step k0, `PLMSBase.mis_merge_step`)."""
    if not 0 < int(S) <= int(ddpm_timesteps):
        raise ValueError(f"S must be in [1, {ddpm_timesteps}], got {S}")
    steps = schedule_steps(S, ddpm_timesteps)
    if int(max_batch) <= 0:
        raise ValueError(f"max_batch must be positive, got {max_batch}")
    if not requests:
        raise ValueError("no requests")
    plans, hw, ctx_len = [], None, None
    for j, req in enumerate(requests):
        if req.S is not None and int(req.S) != int(S):
            raise ValueError(f"request {j}: S={req.S} differs from the call's S={S}")
        if req.mask is not None or req.x0 is not None:
            raise ValueError(f"request {j}: mask / x0 inpainting is not supported by the request drivers; use "
                             "repaint_mask with x_init or init_image")
        multi = isinstance(req.input, (list, tuple))
        kind = SAMPLERS.get(req.sampler)
        if kind is None:
            raise ValueError(f"request {j}: unknown sampler {req.sampler!r} (have {', '.join(SAMPLERS)})")
        if req.output not in OUTPUTS:
            raise ValueError(f"request {j}: unknown output {req.output!r} (have {', '.join(OUTPUTS)})")
        if not req.eta >= 0:
            raise ValueError(f"request {j}: eta={req.eta} must be >= 0")
        if req.eta != 0 and not kind.eta_allowed:
            names = " / ".join(f"sampler={n!r}" for n, k in SAMPLERS.items() if k.eta_allowed)
            raise ValueError(f"request {j}: eta={req.eta} needs {names} ({kind.title} is deterministic, eta = 0)")
        if not kind.multi_instance and (multi or req.mis != 0):
            names = " / ".join(k.title for k in SAMPLERS.values() if k.multi_instance)
            raise ValueError(f"request {j}: {kind.title} takes one input dict with mis = 0; the Multi-instance Sampler "
                             f"(input list, mis) is {names} only")
        if req.seed is not None and not 0 <= int(req.seed) < 1 << 64:
            raise ValueError(f"request {j}: seed {req.seed} outside [0, 2^64)")
        if not multi and req.mis != 0:
            raise ValueError(f"request {j}: mis={req.mis} needs the input list [global, inst_1 .. inst_n]; "
                             "a single input dict runs plain PLMS (mis = 0)")
        if not 0 <= req.mis <= 1:
            raise ValueError(f"request {j}: mis={req.mis} outside [0, 1]")
        ins = _inputs_of(req)
        if not ins:
            raise ValueError(f"request {j}: empty input list")
        shapes = {tuple(i["x"].shape) for i in ins if i.get("x") is not None}
        if req.shape is not None:
            shapes.add(tuple(req.shape))
        if len(shapes) != 1:
            raise ValueError(f"request {j}: latent shapes {sorted(shapes)} (give `shape` or one x shape for every input)")
        shape = shapes.pop()
        if len(shape) != 4:
            raise ValueError(f"request {j}: latent shape {shape} is not (B, C, H, W)")
        if hw is None:
            hw = shape[2:]
        elif shape[2:] != hw:
            raise ValueError(f"request {j}: latent {shape[2]}x{shape[3]} differs from {hw[0]}x{hw[1]} of request 0")
        for t in [i["context"] for i in ins] + ([req.uc] if req.uc is not None else []):
            if ctx_len is None:
                ctx_len = t.shape[1]
            elif t.shape[1] != ctx_len:
                raise ValueError(f"request {j}: context length {t.shape[1]} differs from {ctx_len}")
        if req.x_init is not None and req.init_image is not None:
            raise ValueError(f"request {j}: x_init and init_image are exclusive (give the latent or the image)")
        try:
            k0 = check_init(steps, shape, req.x_init, req.strength, image=req.init_image is not None,
                            needs="x_init or init_image")
        except ValueError as e:
            raise ValueError(f"request {j}: {e}") from None
        if req.init_image is not None:
            im = req.init_image
            if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8:
                raise ValueError(f"request {j}: init_image must be a uint8 tensor, got "
                                 f"{getattr(im, 'dtype', type(im).__name__)}")
            want = (8 * shape[2], 8 * shape[3], 3)
            if im.dim() != 4 or im.shape[0] not in (1, shape[0]) or tuple(im.shape[1:]) != want:
                raise ValueError(f"request {j}: init_image of shape {tuple(im.shape)} does not fit the latent {shape} "
                                 f"(want (1 or B, {want[0]}, {want[1]}, 3): 8x the latent, RGB)")
        if req.repaint_mask is not None:
            m = req.repaint_mask
            if not isinstance(m, torch.Tensor) or m.dtype not in (torch.bool, torch.uint8):
                raise ValueError(f"request {j}: repaint_mask must be a bool or uint8 tensor, got "
                                 f"{getattr(m, 'dtype', type(m).__name__)}")
            want = (8 * shape[2], 8 * shape[3])
            if m.dim() != 3 or m.shape[0] not in (1, shape[0]) or tuple(m.shape[1:]) != want:
                raise ValueError(f"request {j}: repaint_mask of shape {tuple(m.shape)} does not fit the latent {shape} "
                                 f"(want (1 or B, {want[0]}, {want[1]}): 8x the latent)")
            if req.x_init is None and req.init_image is None:
                raise ValueError(f"request {j}: repaint_mask needs x_init or init_image (the source of the kept region)")
        img2img = req.x_init is not None or req.init_image is not None
        plans.append(RequestPlan.of(len(ins), req.mis if multi else None, steps, k0, img2img, shape[0],
                                    req.uc is not None and req.guidance_scale != 1))
    return plans


class _RequestState(SamplingRun):
    """One request being sampled by `sample_requests` or `SamplingEngine`: its `SamplingRun` on its sampler kind with
    `make_schedule(S)` (and the request's eta) and its seed, and what the model was when the request was admitted.
    Both drivers evaluate a request the same way: `begin`, one forward of its trajectories at `fuser_scale()` and
    `conv_flag(...)` (`evaluate`), `advance` with the eps; after the last step `finish` returns its latent.  An
    `init_image` request's x_init is set by `encode_init_images` before `start`."""

    def __init__(self, req: Request, plan: RequestPlan, S: int, model, diffusion):
        base = SAMPLERS[req.sampler](diffusion, model)
        base.make_schedule(ddim_num_steps=int(S), ddim_eta=float(req.eta))
        base.seed = resolve_seed(base.noisy() or req.x_init is not None or req.init_image is not None, req.seed)
        ins = _inputs_of(req)
        x = next((i["x"] for i in ins if i.get("x") is not None), None)
        shape = tuple(x.shape) if x is not None else tuple(req.shape)
        steps = len(base.ddim_timesteps)
        alphas = req.alpha_generator_func(steps) if req.alpha_generator_func is not None else None
        super().__init__(base, list(ins), shape, plan, req.guidance_scale, alphas, req.x_init)
        self.req = req
        self.scale = 0.0  # without an alpha schedule: the model's fuser scale at admission
        if self.alphas is None:
            fusers = [m for m in model.modules() if isinstance(m, GatedSelfAttentionDense)]
            self.scale = float(fusers[0].scale) if fusers else 0.0
            if any(float(f.scale) != self.scale for f in fusers):
                raise ValueError("requests without an alpha_generator_func run at the model's fuser scale, "
                                 "which differs between fusers")
        self.restored = bool(getattr(model, "_first_conv_restored", False))
        # uncond inputs: the null grounding tokens of the request's batch (UNetModel.object_kv(None) uses the batch
        # the grounding tokenizer input was last prepared with, which serves batch 1 and that batch)
        gti = getattr(model, "grounding_tokenizer_input", None)
        own = gti is None or not getattr(gti, "set", False) or gti.batch in (1, plan.images)
        self.null_input = None if own else gti.get_null_input(batch=plan.images)
        self.group = (self.shape[2:], ins[0]["context"].shape[1])
        self.reached_zero = False

    def start(self):
        if self.req.init_image is not None and self.x_init is None:
            raise RuntimeError("an init_image request starts after `encode_init_images`")
        if self.req.repaint_mask is not None:
            self.keep = keep_mask(self.req.repaint_mask.to(self.base.device))
        super().start()

    def images(self) -> int:
        """Images the request puts into an evaluation before its merge."""
        return self.plan.trajectories * self.plan.rows()

    def inputs(self) -> List[dict]:
        """Every input dict the request's forwards use: its trajectories and its uncond branch."""
        ins = list(self.ins)
        if self.plan.cfg:
            ins.append(dict(context=self.req.uc, grounding_input=self.null_input))
        return ins

    def fuser_scale(self) -> float:
        """Fuser scale of step i.  Sets `reached_zero` from the first alpha 0 on: there the request's own sampler
        swaps in the SD1.5 conv (PLMSBase._set_alpha)."""
        if self.alphas is None:
            return self.scale
        alpha = float(self.alphas[self.i])
        self.reached_zero |= alpha == 0
        return alpha

    def conv_flag(self, sd_conv: bool) -> bool:
        """Whether the request's images take the SD1.5 conv: the model had it at admission, or the request reached
        alpha 0 and `sd_conv` says the model has that conv to give."""
        return self.restored or (self.reached_zero and sd_conv)

    @staticmethod
    def evaluate(model, states: Sequence[_RequestState], forwards: Sequence[Tuple[List[Tuple[int, int]], Optional[int]]],
                 scales: Sequence[float], flags: Sequence[bool]):
        """One UNet evaluation of the trajectories of `forwards`, one forward per (chunk of (request, trajectory) slots,
        padded size), each request's images at its fuser scale and conv flag: {(request, trajectory): (e_c, e_u|None)}.
        A chunk with a padded size is filled up to it with copies of its last input (same context and grounding, so
        its hoisted tensors come from the caches) with a zero latent, fuser scale 0 and the model's own conv; their
        outputs are dropped."""
        out = {}
        for chunk, padded in forwards:
            inputs, sc, rs = [], [], []
            for r, k in chunk:
                st = states[r]
                tr = st.trajs[k]
                inputs.append(tr.input)
                if st.plan.cfg:
                    inputs.append(dict(x=tr.input["x"], timesteps=tr.input["timesteps"], context=st.req.uc,
                                       grounding_input=st.null_input))
                n = 2 if st.plan.cfg else 1
                sc += [scales[r]] * n
                rs += [flags[r]] * n
            if padded is not None:
                last = inputs[-1]
                pad = dict(last, x=torch.zeros_like(last["x"]))
                n_pad = (padded - sum(i["x"].shape[0] for i in inputs)) // last["x"].shape[0]
                inputs += [pad] * n_pad
                sc += [0.0] * n_pad
                rs += [False] * n_pad
            outs = model.forward_batched(inputs, scales=sc, restored=rs)
            j = 0
            for r, k in chunk:
                if states[r].plan.cfg:
                    out[(r, k)] = (outs[j], outs[j + 1])
                    j += 2
                else:
                    out[(r, k)] = (outs[j], None)
                    j += 1
        return out

    @staticmethod
    def encode_init_images(states: Sequence[_RequestState], autoencoder, max_encode_batch: int) -> None:
        """The x_init of every `init_image` request among `states`, encoded together by `encode_images` on the
        requests' device, each with its own seed."""
        enc = [st for st in states if st.req.init_image is not None]
        if enc:
            zs = encode_images(autoencoder, [st.req.init_image.to(st.base.device) for st in enc],
                               [st.base.seed for st in enc], max_encode_batch)
            for st, z in zip(enc, zs):
                st.x_init = z

    @staticmethod
    @contextmanager
    def cache_bounds(model, hoist: int, cat: int, graph_pool=None):
        """Within the block, the model's hoisted-tensor caches hold at least `hoist` text / object K/V entries and `cat`
        concatenations and, if given, new CUDA-graph captures use `graph_pool`; afterwards the model has its own
        values again."""
        bounds = {"hoist_cache_entries": max(hoist, getattr(model, "hoist_cache_entries", 0)),
                  "cat_cache_entries": max(cat, getattr(model, "cat_cache_entries", 0))}
        if graph_pool is not None:
            bounds["graph_pool"] = graph_pool
        saved = {k: model.__dict__[k] for k in bounds if k in model.__dict__}
        for k, v in bounds.items():
            setattr(model, k, v)
        try:
            yield
        finally:
            for k in bounds:
                if k in saved:
                    setattr(model, k, saved[k])
                else:
                    delattr(model, k)


def keep_mask(repaint_mask: torch.Tensor) -> torch.Tensor:
    """The latent keep mask of a pixel repaint mask (Bm, 8H, 8W): uint8 (Bm, H, W), 1 where no pixel of the cell's 8x8
    block is to be repainted."""
    bm, h8, w8 = repaint_mask.shape
    rep = (repaint_mask != 0).view(bm, h8 // 8, 8, w8 // 8, 8).any(4).any(2)
    return (~rep).to(torch.uint8)


def paste_back(req: Request, image: torch.Tensor) -> torch.Tensor:
    """The image of a finished request: for an inpainting request started from `init_image`, the decoded `image`
    (B, 8H, 8W, 3) inside its repaint mask and the source's bytes outside it, out[b, y, x] = repaint[b % Bm, y, x] ?
    image[b, y, x] : init_image[b % Bi, y, x]; any other request's image as it is."""
    if req.repaint_mask is None or req.init_image is None:
        return image
    rep = req.repaint_mask.to(image.device) != 0
    return torch.where(rep[..., None], image, req.init_image.to(image.device))


def check_decode(requests: Sequence[Request], autoencoder, max_decode_batch: int, max_encode_batch: int = 8) -> None:
    """The first-stage settings of a driver for `requests`: image outputs and image inputs need an autoencoder."""
    if int(max_decode_batch) <= 0:
        raise ValueError(f"max_decode_batch must be positive, got {max_decode_batch}")
    if int(max_encode_batch) <= 0:
        raise ValueError(f"max_encode_batch must be positive, got {max_encode_batch}")
    if autoencoder is None:
        for j, req in enumerate(requests):
            if req.output == "image":
                raise ValueError(f"request {j}: output='image' needs the driver's autoencoder (autoencoder=None)")
            if req.init_image is not None:
                raise ValueError(f"request {j}: init_image needs the driver's autoencoder (autoencoder=None)")


def _by_size(tensors: Sequence[torch.Tensor], max_batch: int, fn) -> List[torch.Tensor]:
    """fn over `tensors` (each (B_j, ...)) together: the tensors of one size are concatenated in order and passed in
    chunks of at most `max_batch` images as fn(chunk, [(j, b)] of its images); one output per tensor, in order."""
    out: List[Optional[torch.Tensor]] = [None] * len(tensors)
    by_size: Dict[tuple, List[int]] = {}
    for j, t in enumerate(tensors):
        by_size.setdefault(tuple(t.shape[1:]), []).append(j)
    m = int(max_batch)
    for js in by_size.values():
        x = tensors[js[0]] if len(js) == 1 else torch.cat([tensors[j] for j in js])
        owners = [(j, b) for j in js for b in range(tensors[j].shape[0])]
        parts = [fn(x[s:s + m], owners[s:s + m]) for s in range(0, x.shape[0], m)]
        y = parts[0] if len(parts) == 1 else torch.cat(parts)
        start = 0
        for j in js:
            out[j] = y[start:start + tensors[j].shape[0]]
            start += tensors[j].shape[0]
    return out


def encode_images(autoencoder, images: Sequence[torch.Tensor], seeds: Sequence[int],
                  max_encode_batch: int) -> List[torch.Tensor]:
    """The latents of `images` (each uint8 (B_j, H, W, 3), on one device), encoded together: the images of one size
    are concatenated in order and run through the autoencoder in chunks of at most `max_encode_batch` images, image b of
    entry j with seed seeds[j] and index b.  One fp32 (B_j, 4, H/8, W/8) latent per entry, in order, each equal to
    `autoencoder.encode_images(images[j], seed=seeds[j])` (bit for bit in batch-invariant mode)."""
    return _by_size(images, max_encode_batch, lambda x, owners: autoencoder._encode_images(
        x, [int(seeds[j]) for j, _ in owners], [b for _, b in owners]))


def decode_latents(autoencoder, latents: Sequence[torch.Tensor], max_decode_batch: int) -> List[torch.Tensor]:
    """The images of `latents` (each (B_j, 4, h, w)), decoded together: the latents of one size are concatenated in
    order and run through `autoencoder.decode_images` in chunks of at most `max_decode_batch` images; one uint8
    (B_j, 8h, 8w, 3) tensor per latent, in order."""
    return _by_size(latents, max_decode_batch, lambda z, _: autoencoder.decode_images(z))


@torch.no_grad()
def sample_requests(model, diffusion, requests: Sequence[Union[Request, Dict]], S: int, *,
                    max_batch: int = 32, autoencoder=None, max_decode_batch: int = 8,
                    max_encode_batch: int = 8) -> List[torch.Tensor]:
    """Sample every request in `requests` (Request objects or dicts of its fields) with S steps of its sampler; returns
    one latent per request, in order, or for an `output="image"` request its uint8 (B, 8H, 8W, 3) image.  `max_batch`
    bounds the images of one UNet forward.  After the last step the latents of the image requests are decoded
    together by `autoencoder` (an `AutoencoderKL`, required when a request asks for an image), at most
    `max_decode_batch` images per decoder forward (`decode_latents`).  Before the first step the `init_image` requests'
    images are encoded together by `autoencoder`, at most `max_encode_batch` images per encoder forward
    (`encode_images`).

    The per-image fuser scales are those `utils.model.set_alpha_scale` sets (every gated fuser at the request's
    alpha), and the model is left with that function's result for the last alpha of the last request that has an
    alpha schedule.  Uncond images take the null grounding tokens of their own batch; where the grounding tokenizer
    input was last prepared at a batch other than 1 and the request's, the request's own `sample()` would raise
    instead ("grounding batch ... does not match latent batch")."""
    from ....utils.model import set_alpha_scale
    reqs = [r if isinstance(r, Request) else Request(**r) for r in requests]
    plans = check_requests(reqs, S, max_batch, diffusion.num_timesteps)
    check_decode(reqs, autoencoder, max_decode_batch, max_encode_batch)
    states = [_RequestState(r, p, S, model, diffusion) for r, p in zip(reqs, plans)]
    _RequestState.encode_init_images(states, autoencoder, max_encode_batch)
    for st in states:
        st.start()
    steps = states[0].steps
    # the model's hoisted-tensor caches must hold every input and every chunk combination of the run, or each
    # forward recomputes its text / object K/V: raised for the run.  Image-to-image requests of a `corrector_first`
    # kind (PLMS) take the corrector's evaluation of their first step in forwards of their own at their start step.
    chunks = {tuple(c) for i in range(steps) for c in plan_step(plans, i, max_batch)}
    for k0 in {p.k0 for p in plans if p.k0 > 0}:
        slots = [(r, k) for r, p in enumerate(plans) if p.k0 == k0 and states[r].base.corrector_first
                 for k in range(p.live(k0))]
        chunks |= {tuple(c) for c in plan_chunks(slots, plans, max_batch)}
    try:
        with _RequestState.cache_bounds(model, sum(p.trajectories + 2 for p in plans) + 8, 2 * len(chunks) + 2):
            for step in range(steps):
                live = [r for r, p in enumerate(plans) if p.k0 <= step]  # image-to-image requests join at k0
                scales, flags = [0.0] * len(states), [False] * len(states)
                for r in live:
                    st = states[r]
                    st.begin()
                    zero = st.reached_zero
                    scales[r] = st.fuser_scale()
                    if st.reached_zero and not zero:
                        model.restore_first_conv_from_SD()  # the swap a run of this request makes here
                sd_conv = bool(getattr(model, "_first_conv_restored", False))
                for r in live:
                    flags[r] = states[r].conv_flag(sd_conv)
                todo = live
                while todo:  # every request's step, then the corrector's evaluation of a first PLMS step
                    slots = [(r, k) for r in todo for k in range(len(states[r].trajs))]
                    forwards = [(c, None) for c in plan_chunks(slots, plans, max_batch)]
                    evals = _RequestState.evaluate(model, states, forwards, scales, flags)
                    for r in todo:
                        states[r].advance([evals[(r, k)] for k in range(len(states[r].trajs))])
                    todo = [r for r in todo if states[r].pending is not None]
    finally:
        model.trim_hoisted()  # the run's concatenations (hundreds of MB each) do not outlive it
    latents = [st.finish() for st in states]
    # the model's fuser scale as a sequential run leaves it: the last alpha of the last request that sets one
    for st in reversed(states):
        if st.alphas is not None:
            set_alpha_scale(model, st.alphas[-1])
            break
    images = [j for j, r in enumerate(reqs) if r.output == "image"]
    if images:
        for j, img in zip(images, decode_latents(autoencoder, [latents[j] for j in images], max_decode_batch)):
            latents[j] = paste_back(reqs[j], img)
    return latents
