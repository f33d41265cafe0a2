"""Many independent sampling requests advanced in lock step (not a reference module).

A deployment that gets one layout per user would otherwise run one `sample()` call per request: every forward
then has the batch of that one request (cond + uncond of one image: 512 GEMM rows at the 16x16 level against
128-row tiles).  `sample_requests` evaluates, at every step, the live trajectories of all requests together in
`forward_batched` chunks of up to `max_batch` images, each image with its own request's fuser scale (alpha
schedule) and first-conv state.  Per request the arithmetic is that of its own sampler: the history and the
PLMS updates are `PLMSBase._step_predict` / `_step_finish` on its own trajectories with its own guidance scale,
and a Multi-instance request merges its latents with `ops.latent_mean` at its own step int(steps * mis), where
steps is the length of the PLMS schedule (`schedule_steps`: S + 1 for some S, e.g. 31 for S = 30), as there.
That per-request machinery is `_RequestState`, which `SamplingEngine` (engine.py) drives too: `sample_requests` is
the lock-step driver on top of it.

Contract: each returned latent equals, within floating-point tolerance, what `PLMSSampler.sample()` (input dict,
mis = 0) or `PLMSSamplerInst.sample()` (input list [global, instance_1 .. instance_n]) returns for that request
alone on the model in the state it had when `sample_requests` was called.  Afterwards the model's fuser scale and
first-conv swap are what a sequential run of the same requests would leave.
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .... import ops
from ...modules.attention import GatedSelfAttentionDense
from ...modules.diffusionmodules.util import make_ddim_timesteps
from ._plms_common import PLMSBase, Trajectory


@dataclass
class Request:
    """One sampling request.  `input`: the dict `PLMSSampler.sample` takes, or the list [global, inst_1 .. inst_n]
    of `PLMSSamplerInst.sample`; `shape`: (B, 4, H, W) of its latent (may be omitted when input x is given);
    `mis`: the Multi-instance fraction (list inputs only).  `S`: the request's step count; `sample_requests` takes it
    from the call (S, if given, must equal it), `SamplingEngine` requires it.  `mask` / `x0` (inpainting) are not
    supported and raise."""
    input: Union[dict, List[dict]]
    uc: Optional[torch.Tensor] = None
    guidance_scale: float = 1.0
    alpha_generator_func: Optional[Callable[[int], List[float]]] = None
    mis: float = 0.0
    shape: Optional[Tuple[int, ...]] = None
    S: Optional[int] = None
    mask: Optional[torch.Tensor] = None
    x0: Optional[torch.Tensor] = None


@dataclass(frozen=True)
class RequestPlan:
    """What the step planner needs of a request: trajectories before the merge (1 for plain PLMS), the step
    before which they merge (None: never), images per trajectory and whether it evaluates cond + uncond."""
    trajectories: int
    merge_step: Optional[int]
    images: int
    cfg: bool

    def live(self, step: int) -> int:
        """Trajectories evaluated at `step`."""
        return self.trajectories if self.merge_step is not None and step < self.merge_step else 1

    def rows(self) -> int:
        """Images one trajectory puts into a forward."""
        return self.images * (2 if self.cfg else 1)


def plan_chunks(slots: Sequence[Tuple[int, int]], plans: Sequence[RequestPlan], max_batch: int) -> List[List[Tuple[int, int]]]:
    """Split (request, trajectory) slots, in order, into forward chunks of at most `max_batch` images.  A
    trajectory's cond and uncond images stay in one chunk; a trajectory larger than `max_batch` gets a chunk
    of its own."""
    chunks, cur, used = [], [], 0
    for r, k in slots:
        n = plans[r].rows()
        if cur and used + n > max_batch:
            chunks.append(cur)
            cur, used = [], 0
        cur.append((r, k))
        used += n
    if cur:
        chunks.append(cur)
    return chunks


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
    step count S, the latent height x width and the context length; mask / x0 inpainting is not supported.
    A Multi-instance request merges before step int(schedule_steps(S) * mis), as PLMSSamplerInst does."""
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
            raise ValueError(f"request {j}: mask / x0 inpainting is not supported by sample_requests")
        multi = isinstance(req.input, (list, tuple))
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
        cfg = req.uc is not None and req.guidance_scale != 1
        plans.append(RequestPlan(len(ins), int(steps * req.mis) if multi else None, shape[0], cfg))
    return plans


class _RequestState:
    """One request being sampled by `sample_requests` or `SamplingEngine`: its plan and its own PLMS schedule
    (`make_schedule(S)`), what the model was when the request was admitted, and, once started, its trajectories and its
    position in the schedule.  Both drivers evaluate a request the same way: `begin`, one forward of its trajectories at
    `fuser_scale()` and `conv_flag(...)`, `advance` with the eps; after the last step `finish` returns its latent."""

    def __init__(self, req: Request, plan: RequestPlan, S: int, model, diffusion):
        self.req, self.plan = req, plan
        self.base = PLMSBase(diffusion, model)
        self.base.make_schedule(ddim_num_steps=int(S))
        self.time_range = np.flip(self.base.ddim_timesteps)
        self.steps = len(self.time_range)
        self.alphas = req.alpha_generator_func(self.steps) if req.alpha_generator_func is not None else None
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
        ins = _inputs_of(req)
        x = next((i["x"] for i in ins if i.get("x") is not None), None)
        self.group = (tuple(x.shape[2:]) if x is not None else tuple(req.shape[2:]), ins[0]["context"].shape[1])
        self.trajs: List[Trajectory] = []
        self.gs = float(req.guidance_scale)
        self.reached_zero = False
        self.i = 0             # current step
        self.pending = None    # predictor state while the corrector's evaluation is due
        self.ts_next = None

    def start(self):
        """The trajectories, when the request starts sampling."""
        ins = _inputs_of(self.req)
        if ins[0].get("x") is None:  # as the samplers: one noise tensor shared by every trajectory
            img = torch.randn(tuple(self.req.shape), device=self.base.device)
            for inp in ins:
                inp["x"] = img
        self.trajs = [Trajectory(inp) for inp in ins]

    def images(self) -> int:
        """Images the request puts into an evaluation before its merge."""
        return self.plan.trajectories * self.plan.rows()

    def inputs(self) -> List[dict]:
        """Every input dict the request's forwards use: its trajectories and its uncond branch."""
        ins = list(_inputs_of(self.req))
        if self.plan.cfg:
            ins.append(dict(context=self.req.uc, grounding_input=self.null_input))
        return ins

    def merge(self):
        """Multi-instance merge: the global trajectory continues from the mean of the n+1 latents
        (plms_instance.py:135).  A single trajectory is left as it is."""
        if len(self.trajs) > 1:
            xs = [tr.input["x"].float().contiguous() for tr in self.trajs]
            merged = torch.empty_like(xs[0])
            ops.latent_mean(xs, merged)
            self.trajs[0].input["x"] = merged
            self.trajs = self.trajs[:1]

    def begin(self):
        """Before an evaluation: the merge due before step i and the timesteps of step i, unless the evaluation is the
        corrector's of the first PLMS step (the predictor left the inputs at t_next)."""
        if self.pending is None:
            if self.plan.merge_step == self.i:
                self.merge()
            ts, self.ts_next = self.base._timesteps(self.plan.images, self.i, self.time_range)
            for tr in self.trajs:
                tr.input["timesteps"] = ts

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

    def advance(self, evals):
        """Advance by an evaluation's [(e_c, e_u|None)] per trajectory: the predictor of a first PLMS step, which
        leaves `pending` set until the corrector's evaluation, or the corrector or a plain step, which moves to step
        i + 1."""
        index = self.steps - self.i - 1
        pending, self.pending = self.pending, None
        if pending is None:
            self.pending = self.base._step_predict(self.trajs, evals, self.ts_next, index, self.gs)
            if self.pending is not None:
                return
        self.base._step_finish(self.trajs, evals, pending, index, self.gs)
        self.i += 1

    def finish(self) -> torch.Tensor:
        """The latent, after the last step and, for mis = 1, the merge that follows it."""
        if self.plan.merge_step == self.steps:
            self.merge()
        return self.trajs[0].input["x"]

    @staticmethod
    def evaluate(model, states: Sequence[_RequestState], forwards: Sequence[Tuple[List[Tuple[int, int]], Optional[int]]],
                 scales: Sequence[float], flags: Sequence[bool], per_image_conv: bool = False):
        """One UNet evaluation of the trajectories of `forwards`, one forward per (chunk of (request, trajectory) slots,
        padded size), each request's images at its fuser scale and conv flag: {(request, trajectory): (e_c, e_u|None)}.
        A chunk with a padded size is filled up to it with copies of its last input (same context and grounding, so
        its hoisted tensors come from the caches) with a zero latent, fuser scale 0 and the model's own conv; their
        outputs are dropped.  per_image_conv: see UNetModel.forward_batched."""
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
            outs = model.forward_batched(inputs, scales=sc, restored=rs, per_image_conv=per_image_conv)
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


@torch.no_grad()
def sample_requests(model, diffusion, requests: Sequence[Union[Request, Dict]], S: int, *,
                    max_batch: int = 32) -> List[torch.Tensor]:
    """Sample every request in `requests` (Request objects or dicts of its fields) with S PLMS steps; returns one
    latent per request, in order.  `max_batch` bounds the images of one UNet forward.

    The per-image fuser scales are those `utils.model.set_alpha_scale` sets (every gated fuser at the request's
    alpha), and the model is left with that function's result for the last alpha of the last request that has an
    alpha schedule.  Uncond images take the null grounding tokens of their own batch; where the grounding tokenizer
    input was last prepared at a batch other than 1 and the request's, the request's own `sample()` would raise
    instead ("grounding batch ... does not match latent batch")."""
    from ....utils.model import set_alpha_scale
    reqs = [r if isinstance(r, Request) else Request(**r) for r in requests]
    plans = check_requests(reqs, S, max_batch, diffusion.num_timesteps)
    states = [_RequestState(r, p, S, model, diffusion) for r, p in zip(reqs, plans)]
    for st in states:
        st.start()
    steps = states[0].steps
    # the model's hoisted-tensor caches must hold every input and every chunk combination of the run, or each
    # forward recomputes its text / object K/V: raised for the run
    chunks = {tuple(c) for i in range(steps) for c in plan_step(plans, i, max_batch)}
    try:
        with _RequestState.cache_bounds(model, sum(p.trajectories + 2 for p in plans) + 8, 2 * len(chunks) + 2):
            for _ in range(steps):
                scales = []
                for st in states:
                    st.begin()
                    zero = st.reached_zero
                    scales.append(st.fuser_scale())
                    if st.reached_zero and not zero:
                        model.restore_first_conv_from_SD()  # the swap a run of this request makes here
                sd_conv = bool(getattr(model, "_first_conv_restored", False))
                flags = [st.conv_flag(sd_conv) for st in states]
                todo = range(len(states))
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
    return latents
