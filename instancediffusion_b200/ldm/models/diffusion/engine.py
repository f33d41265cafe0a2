"""Continuous batching of sampling requests (not a reference module).

`sample_requests` advances a fixed set of requests in lock step: every request starts at step 0 and the call returns
when the slowest one finishes.  `SamplingEngine` lets requests join and leave between steps instead:

    engine = SamplingEngine(model, diffusion, max_batch=32)
    ticket = engine.submit(request)      # Request of batched.py with its own step count request.S
    done = engine.step()                 # one tick: {ticket: latent} of the requests that finished in it
    done = engine.drain()                # tick until nothing is queued or live

A tick gives every live trajectory exactly one UNet evaluation: the one at t of its current step or, for a request
in the Euler predictor of its first PLMS step, the corrector's evaluation at t_next (so the corrector rides in the
next tick with everyone else).  A PLMS request therefore retires after schedule_steps(S) + 1 ticks, a DDIM request
(one evaluation per step) after schedule_steps(S).  Each request is a `batched._RequestState`, the per-request sampling
state that `sample_requests` drives too: its own schedule (`make_schedule(S)` of `PLMSBase`, or of `DDIMBase` with its
eta and seed), its sampler's arithmetic (`_step_predict` / `_step_finish`) and its Multi-instance merge before step
int(schedule_steps(S) * mis), after the last one for mis = 1.  PLMS and DDIM requests of one latent size and context
length share forwards.  The engine adds admission, the grouping of a tick's forwards and retirement.

The evaluations of a tick are grouped by (latent H x W, context length) in admission order, split into forwards of
at most `max_batch` images by `plan_chunks`, and each forward is padded to the smallest of `buckets` that holds it.
The forwards choose the fuser scale and the input conv per image on the device (`UNetModel.forward_batched(scales=,
per_image_conv=True)`), so the captured CUDA graphs do not depend on the composition of the batch: per latent size,
context length, mask presence and fuser state (off / per image / one common scale) there are at most len(buckets).
The engine never calls set_alpha_scale or swaps the model's first conv.

Contract: each returned latent equals, within floating-point tolerance, what the request's own
`PLMSSampler.sample()` / `PLMSSamplerInst.sample()` / `DDIMSampler.sample(eta=, seed=)` returns when it runs alone on
the model in the state it had at `submit`, whatever else is live and whenever the request arrived.
"""
from __future__ import annotations

from collections import deque
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from .batched import Request, RequestPlan, _RequestState, check_requests, plan_chunks


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
        self._queue: deque = deque()                     # (ticket, state), in submission order
        self._live: Dict[int, _RequestState] = {}        # ticket -> state, in admission order
        self._next = 0
        self.graphs_captured = 0
        self.forwards = 0        # UNet forwards run
        self.padded_images = 0   # padding images among them

    @property
    def queued(self) -> List[int]:
        return [t for t, _ in self._queue]

    @property
    def live(self) -> List[int]:
        return list(self._live)

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
        st = _RequestState(req, plan, int(req.S), self.model, self.diffusion)
        ticket, self._next = self._next, self._next + 1
        self._queue.append((ticket, st))
        return ticket

    def drain(self) -> Dict[int, torch.Tensor]:
        """Tick until nothing is queued or live; the latents of every request that finished meanwhile."""
        done = {}
        while self._queue or self._live:
            done.update(self.step())
        return done

    @torch.no_grad()
    def step(self) -> Dict[int, torch.Tensor]:
        """One tick: admit, evaluate every live trajectory once, advance; {ticket: latent} of the finished requests."""
        live_images = sum(st.images() for st in self._live.values())
        while self._queue and live_images + self._queue[0][1].images() <= self.max_live_images:
            ticket, st = self._queue.popleft()
            st.start()
            self._live[ticket] = st
            live_images += st.images()
        if not self._live:
            return {}
        states = list(self._live.values())
        sd_conv = getattr(self.model, "first_conv_restorable", True)
        scales, flags = [], []
        for st in states:
            st.begin()
            scales.append(st.fuser_scale())
            flags.append(st.conv_flag(sd_conv))
        slots = [(r, k) for r, st in enumerate(states) for k in range(len(st.trajs))]
        forwards = plan_forwards(slots, [st.plan for st in states], [st.group for st in states], self.max_batch,
                                 self.buckets)
        evals = self._run(states, forwards, scales, flags)

        done = {}
        for r, (ticket, st) in enumerate(list(self._live.items())):
            st.advance([evals[(r, k)] for k in range(len(st.trajs))])
            if st.i == st.steps:
                done[ticket] = st.finish()
        finished = [self._live.pop(t) for t in done]
        if finished:
            keep = [i for st in list(self._live.values()) + [st for _, st in self._queue] for i in st.inputs()]
            self.model.drop_hoisted([i for st in finished for i in st.inputs()], keep)
        return done

    def _run(self, states, forwards, scales, flags):
        """The forwards of a tick, with the model's hoisted-tensor cache bounds raised as far as the live set needs
        and, if shared, the engine's graph pool; concatenations of chunks this tick did not use are dropped."""
        model = self.model
        if self.share_graph_pool and self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()
        n_graphs = len(model._graphs)
        with _RequestState.cache_bounds(model, sum(st.plan.trajectories + 1 for st in states) + 8,
                                        len(model._cat_cache) + len(forwards) + 1, self._pool):
            evals = _RequestState.evaluate(model, states, forwards, scales, flags, per_image_conv=True)
        self.graphs_captured += len(model._graphs) - n_graphs
        model.trim_concats(len(forwards))
        self.forwards += len(forwards)
        for chunk, padded in forwards:
            if padded is not None:
                self.padded_images += padded - sum(states[r].plan.rows() for r, _ in chunk)
        return evals
