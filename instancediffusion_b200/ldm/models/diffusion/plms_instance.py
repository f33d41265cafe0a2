"""PLMSSamplerInst, the Multi-instance Sampler -- drop-in for ldm/models/diffusion/plms_instance.py.

For the first int(S*mis) steps every instance is denoised on its own trajectory (its own phrase as
context and a single-instance grounding input) next to the global one; the latents are then
averaged (plms_instance.py:135) and the remaining steps run on the merged global latent.
The reference walks the n+1 trajectories sequentially; they are independent until the merge, so
here each step evaluates all of them (cond and uncond) in one batched UNet forward.
An image-to-image run (x_init) starting at or after the merge step runs the global trajectory alone
(PLMSBase.mis_merge_step)."""
import os

import numpy as np
import torch

from .... import ops
from ._plms_common import PLMSBase, Trajectory


class PLMSSamplerInst(PLMSBase):
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None, mis=0.0):
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)
        self.mis = mis
        # upper bound on trajectories evaluated in one batched forward (memory knob)
        self.max_group = int(os.environ.get("IDIFF_MIS_GROUP", "16"))

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, x_init=None, strength=1.0,
               seed=None):
        """plms_instance.py:58-63; x_init / strength / seed start image-to-image sampling as in PLMSSampler.sample,
        every trajectory from the same start latent."""
        self.make_schedule(ddim_num_steps=S)
        k0, x_start = self.init_run(shape, x_init, strength, seed)
        if x_start is not None:
            for inp in input:
                inp["x"] = x_start
        return self.plms_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, k0=k0,
                                  img2img=x_start is not None)

    @torch.no_grad()
    def plms_sampling(self, shape, input_all, uc=None, guidance_scale=1, mask=None, x0=None, k0=0, img2img=False):
        """plms_instance.py:65-158, from step k0 (image-to-image) on."""
        b = shape[0]
        if input_all[0]["x"] is None:
            img = torch.randn(shape, device=self.device)
            for inp in input_all:
                inp["x"] = img
        time_range = np.flip(self.ddim_timesteps)
        total_steps = self.ddim_timesteps.shape[0]
        alphas = self.alpha_generator_func(len(time_range)) if self.alpha_generator_func is not None else None
        mis_step = self.mis_merge_step(total_steps, self.mis, k0, img2img)

        trajs = [Trajectory(inp) for inp in input_all]
        glob = trajs[0]
        if mis_step is not None:
            for i in range(k0, mis_step):
                if alphas is not None:
                    self._set_alpha(alphas[i])
                ts, ts_next = self._timesteps(b, i, time_range)
                for g in range(0, len(trajs), self.max_group):
                    self._step(trajs[g:g + self.max_group], ts, ts_next, total_steps - i - 1, uc, guidance_scale)

            # merge: mean over the n+1 latents (the reference's default branch, :135)
            xs = [tr.input["x"].float().contiguous() for tr in trajs]
            merged = torch.empty_like(xs[0])
            ops.latent_mean(xs, merged)
            glob.input["x"] = merged

        for i in range(k0 if mis_step is None else mis_step, len(time_range)):
            if alphas is not None:
                self._set_alpha(alphas[i])
            ts, ts_next = self._timesteps(b, i, time_range)
            self._step([glob], ts, ts_next, total_steps - i - 1, uc, guidance_scale)
        return glob.input["x"]
