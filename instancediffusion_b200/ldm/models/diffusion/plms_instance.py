"""PLMSSamplerInst, the Multi-instance Sampler -- drop-in for ldm/models/diffusion/plms_instance.py.

For the first int(S*mis) steps every instance is denoised on its own trajectory (its own phrase as
context and a single-instance grounding input) next to the global one; the latents are then
averaged (plms_instance.py:135) and the remaining steps run on the merged global latent.
The reference walks the n+1 trajectories sequentially; they are independent until the merge, so
here each step evaluates them (cond and uncond) in batched UNet forwards of at most `max_group`
trajectories (`IDIFF_MIS_GROUP`, default 16): `PLMSBase.sample_loop` with the input list.
An image-to-image run (x_init) starting at or after the merge step runs the global trajectory alone
(PLMSBase.mis_merge_step).  mask / x0 are ignored, as in the reference."""
import os

import torch

from ._plms_common import PLMSBase


class PLMSSamplerInst(PLMSBase):
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None, mis=0.0):
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)
        self.mis = mis
        # upper bound on trajectories evaluated in one batched forward (memory knob)
        self.max_group = int(os.environ.get("IDIFF_MIS_GROUP", "16"))

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, x_init=None, strength=1.0,
               seed=None):
        """plms_instance.py:58-63 on the input list [global, inst_1 .. inst_n]; x_init / strength / seed start
        image-to-image sampling as in PLMSSampler.sample, every trajectory from the same start latent."""
        return self._sample(S, shape, input, uc, guidance_scale, None, None, x_init, strength, seed, mis=self.mis)

    def plms_sampling(self, shape, input_all, uc=None, guidance_scale=1, mask=None, x0=None, k0=0, x_init=None):
        """plms_instance.py:65-158, from step k0 on: `PLMSBase.sample_loop` with the input list."""
        return self.sample_loop(shape, input_all, uc, guidance_scale, k0=k0, x_init=x_init, mis=self.mis)
