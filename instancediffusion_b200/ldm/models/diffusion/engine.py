"""Continuous batching of sampling requests (not a reference module).

`sample_requests` advances a fixed set of requests in lock step: every request starts at step 0 and the call returns
when the slowest one finishes.  `SamplingEngine` lets requests join and leave between steps instead:

    engine = SamplingEngine(model, diffusion, max_batch=32)
    ticket = engine.submit(request)      # Request of batched.py with its own step count request.S
    done = engine.step()                 # one tick: {ticket: latent} of the requests that finished in it
    done = engine.drain()                # tick until nothing is queued or live

A tick gives every live trajectory exactly one UNet evaluation: the one at t of its current step or, for a request
in the Euler predictor of its first PLMS step, the corrector's evaluation at t_next (so the corrector rides in the
next tick with everyone else).  Per request the arithmetic is that of its own sampler, on its own schedule
(`PLMSBase.make_schedule(S)`): history and updates are `PLMSBase._step_predict` / `_step_finish`, and a
Multi-instance request merges before its step int(schedule_steps(S) * mis), after the last one for mis = 1.

The evaluations of a tick are grouped by (latent H x W, context length) in admission order, split into forwards of
at most `max_batch` images by `plan_chunks`, and each forward is padded to the smallest of `buckets` that holds it.
The forwards choose the fuser scale and the input conv per image on the device (`UNetModel.forward_batched(scales=,
per_image_conv=True)`), so the captured CUDA graphs do not depend on the composition of the batch: per latent size,
context length, mask presence and fuser state (off / per image / one common scale) there are at most len(buckets).
The engine never calls set_alpha_scale or swaps the model's first conv.

Contract: each returned latent equals, within floating-point tolerance, what the request's own
`PLMSSampler.sample()` / `PLMSSamplerInst.sample()` returns when it runs alone on the model in the state it had at
`submit`, whatever else is live and whenever the request arrived.
"""
from __future__ import annotations

from collections import deque
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from ...modules.attention import GatedSelfAttentionDense
from ._plms_common import PLMSBase
from .batched import Request, RequestPlan, _State, _evaluate, _inputs_of, check_requests, plan_chunks


def pick_bucket(images: int, unit: int, buckets: Optional[Sequence[int]]) -> Optional[int]:
    """Padded size of a forward of `images` images whose last input has `unit` images: the smallest bucket that
    holds it and that copies of the last input fill exactly.  None: no such bucket (or no buckets): run unpadded."""
    for b in buckets or ():
        if b >= images and (b - images) % unit == 0:
            return b
    return None


def plan_forwards(slots: Sequence[Tuple[int, int]], plans: Sequence[RequestPlan], groups: Sequence[tuple],
                  max_batch: int, buckets: Optional[Sequence[int]]) -> List[Tuple[List[Tuple[int, int]], Optional[int]]]:
    """The forwards of one tick: (request, trajectory) slots grouped by `groups[request]` (latent H x W, context
    length) in order of first appearance, each group split by `plan_chunks`, each chunk with its padded size."""
    by_group: Dict[tuple, list] = {}
    for r, k in slots:
        by_group.setdefault(groups[r], []).append((r, k))
    out = []
    for group_slots in by_group.values():
        for chunk in plan_chunks(group_slots, plans, max_batch):
            images = sum(plans[r].rows() for r, _ in chunk)
            last = plans[chunk[-1][0]]
            out.append((chunk, pick_bucket(images, last.images, buckets)))
    return out


class _Live:
    """A submitted request: its plan, its own schedule and, once admitted, its sampling state and position."""

    def __init__(self, ticket: int, req: Request, plan: RequestPlan, base: PLMSBase, scale: float, restored: bool,
                 null_input, group: tuple):
        self.ticket, self.req, self.plan, self.base = ticket, req, plan, base
        self.time_range = np.flip(base.ddim_timesteps)
        self.steps = len(self.time_range)
        self.scale, self.restored = scale, restored  # fuser scale / first-conv state of the model at submit
        self.null_input, self.group = null_input, group
        self.state: Optional[_State] = None
        self.i = 0               # current step
        self.pending = None      # predictor state while the corrector evaluation is due
        self.ts_next = None

    def images(self) -> int:
        """Images this request puts into a tick's forwards (its trajectories before the merge)."""
        return self.plan.trajectories * self.plan.rows()

    def inputs(self) -> List[dict]:
        """Every input dict the request's forwards use: its trajectories and its uncond branch."""
        ins = list(_inputs_of(self.req))
        if self.plan.cfg:
            ins.append(dict(context=self.req.uc, grounding_input=self.null_input))
        return ins


class SamplingEngine:
    """Step-level scheduler of sampling requests on one model.  `max_batch`: images per UNet forward;
    `max_live_images`: bound of the images of the admitted requests (default 4 * max_batch); `buckets`: the padded
    forward sizes (None: no padding); `share_graph_pool`: capture the graphs of the engine's forwards into one
    memory pool instead of a private pool each (see README)."""

    def __init__(self, model, diffusion, *, max_batch: int = 32, max_live_images: Optional[int] = None,
                 buckets: Optional[Sequence[int]] = (2, 4, 8, 16, 24, 32), share_graph_pool: bool = False):
        if int(max_batch) <= 0:
            raise ValueError(f"max_batch must be positive, got {max_batch}")
        self.model, self.diffusion = model, diffusion
        self.max_batch = int(max_batch)
        self.max_live_images = 4 * self.max_batch if max_live_images is None else int(max_live_images)
        if self.max_live_images <= 0:
            raise ValueError(f"max_live_images must be positive, got {max_live_images}")
        if buckets is not None:
            buckets = tuple(sorted(int(b) for b in buckets))
            if not buckets or buckets[0] <= 0:
                raise ValueError(f"buckets must be positive sizes, got {buckets}")
        self.buckets = buckets
        self.share_graph_pool = bool(share_graph_pool)
        self._pool = None
        self._queue: deque = deque()
        self._live: List[_Live] = []
        self._next = 0
        self.graphs_captured = 0
        self.forwards = 0        # UNet forwards run
        self.padded_images = 0   # padding images among them

    @property
    def queued(self) -> List[int]:
        return [e.ticket for e in self._queue]

    @property
    def live(self) -> List[int]:
        return [e.ticket for e in self._live]

    # --------------------------------------------------------------------------------------------
    def submit(self, request: Union[Request, dict]) -> int:
        """Validate a request and queue it; returns its ticket.  It is admitted FIFO at the start of a later tick,
        when the live images stay within max_live_images."""
        req = request if isinstance(request, Request) else Request(**request)
        if req.S is None:
            raise ValueError("request.S (the request's step count) is required")
        plan = check_requests([req], int(req.S), self.max_batch, self.diffusion.num_timesteps)[0]
        size = plan.trajectories * plan.rows()
        if size > self.max_live_images:
            raise ValueError(f"request of {size} images (trajectories x images x CFG) exceeds max_live_images="
                             f"{self.max_live_images}")
        model = self.model
        scale = 0.0
        if req.alpha_generator_func is None:  # runs at the model's fuser scale, as set when submitted
            fusers = [m for m in model.modules() if isinstance(m, GatedSelfAttentionDense)]
            scale = float(fusers[0].scale) if fusers else 0.0
            if any(float(f.scale) != scale for f in fusers):
                raise ValueError("requests without an alpha_generator_func run at the model's fuser scale, "
                                 "which differs between fusers")
        restored = bool(getattr(model, "_first_conv_restored", False))
        # uncond inputs: the null grounding tokens of the request's batch (as sample_requests)
        gti = getattr(model, "grounding_tokenizer_input", None)
        own = gti is None or not getattr(gti, "set", False) or gti.batch in (1, plan.images)
        null_input = None if own else gti.get_null_input(batch=plan.images)
        ins = _inputs_of(req)
        x = next((i["x"] for i in ins if i.get("x") is not None), None)
        hw = tuple(x.shape[2:]) if x is not None else tuple(req.shape[2:])
        base = PLMSBase(self.diffusion, model)
        base.make_schedule(ddim_num_steps=int(req.S))
        e = _Live(self._next, req, plan, base, scale, restored, null_input, (hw, ins[0]["context"].shape[1]))
        self._next += 1
        self._queue.append(e)
        return e.ticket

    def drain(self) -> Dict[int, torch.Tensor]:
        """Tick until nothing is queued or live; the latents of every request that finished meanwhile."""
        done = {}
        while self._queue or self._live:
            done.update(self.step())
        return done

    @torch.no_grad()
    def step(self) -> Dict[int, torch.Tensor]:
        """One tick: admit, evaluate every live trajectory once, advance; {ticket: latent} of the finished requests."""
        live_images = sum(e.images() for e in self._live)
        while self._queue and live_images + self._queue[0].images() <= self.max_live_images:
            e = self._queue.popleft()
            e.state = _State(e.req, e.plan, e.steps, e.base.device)
            self._live.append(e)
            live_images += e.images()
        if not self._live:
            return {}
        restorable = getattr(self.model, "first_conv_restorable", True)
        scales, restored = [], []
        for e in self._live:
            st = e.state
            if e.pending is None:
                if e.plan.merge_step == e.i and len(st.trajs) > 1:
                    st.merge()
                ts, e.ts_next = e.base._timesteps(e.plan.images, e.i, e.time_range)
                for tr in st.trajs:
                    tr.input["timesteps"] = ts
            alpha = st.alphas[e.i] if st.alphas is not None else e.scale
            if st.alphas is not None and alpha == 0:
                st.reached_zero = True  # the step where its own sampler swaps in the SD1.5 conv
            scales.append(float(alpha))
            restored.append(e.restored or (st.reached_zero and restorable))
        states = [e.state for e in self._live]
        slots = [(r, k) for r, st in enumerate(states) for k in range(len(st.trajs))]
        forwards = plan_forwards(slots, [st.plan for st in states], [e.group for e in self._live], self.max_batch,
                                 self.buckets)
        evals = self._run(states, forwards, scales, restored)

        done, still = {}, []
        for r, e in enumerate(self._live):
            st = e.state
            ev = [evals[(r, k)] for k in range(len(st.trajs))]
            index = e.steps - e.i - 1
            if e.pending is not None:  # the corrector of the first PLMS step
                e.base._step_finish(st.trajs, ev, e.pending, index, st.gs)
                e.pending = None
            else:
                e.pending = e.base._step_predict(st.trajs, ev, e.ts_next, index, st.gs)
                if e.pending is not None:  # the corrector's evaluation at t_next comes next tick
                    still.append(e)
                    continue
                e.base._step_finish(st.trajs, ev, None, index, st.gs)
            e.i += 1
            if e.i < e.steps:
                still.append(e)
                continue
            if e.plan.merge_step == e.steps and len(st.trajs) > 1:  # mis = 1: the merge follows the last step
                st.merge()
            done[e.ticket] = st.trajs[0].input["x"]
        finished = [e for e in self._live if e.ticket in done]
        self._live = still
        if finished:
            keep = [i for e in list(self._live) + list(self._queue) for i in e.inputs()]
            self.model.drop_hoisted([i for e in finished for i in e.inputs()], keep)
        return done

    def _run(self, states, forwards, scales, restored):
        """The forwards of a tick, with the model's hoisted-tensor cache bounds raised as far as the live set needs
        and, if shared, the engine's graph pool; concatenations of chunks this tick did not use are dropped."""
        model = self.model
        n_inputs = sum(len(_inputs_of(st.req)) + 1 for st in states)
        bounds = {"hoist_cache_entries": n_inputs + 8,
                  "cat_cache_entries": len(model._cat_cache) + len(forwards) + 1}
        if self.share_graph_pool:
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            bounds["graph_pool"] = self._pool
        saved = {k: model.__dict__[k] for k in bounds if k in model.__dict__}
        for k, v in bounds.items():
            setattr(model, k, v if k == "graph_pool" else max(v, getattr(model, k, 0)))
        n_graphs = len(model._graphs)
        try:
            evals = _evaluate(model, states, forwards, scales, restored, [e.null_input for e in self._live],
                              per_image_conv=True)
        finally:
            for k in bounds:
                if k in saved:
                    setattr(model, k, saved[k])
                else:
                    delattr(model, k)
        self.graphs_captured += len(model._graphs) - n_graphs
        model.trim_concats(len(forwards))
        self.forwards += len(forwards)
        for chunk, padded in forwards:
            if padded is not None:
                self.padded_images += padded - sum(states[r].plan.rows() for r, _ in chunk)
        return evals
