"""PLMSSampler -- drop-in for ldm/models/diffusion/plms.py (same constructor and `sample`)."""
import numpy as np
import torch

from ._plms_common import PLMSBase, Trajectory


class PLMSSampler(PLMSBase):
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None):
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, x_init=None, strength=1.0,
               seed=None):
        """plms.py:65-70.  x_init (a latent of shape (1 or B, C, H, W)) starts image-to-image sampling: the run takes
        the last int(N * strength) of the N steps from x_init noised to the first of them, the noise keyed by `seed`
        (None: one draw from torch's default CPU generator).  Without x_init this is the reference's sampler."""
        self.make_schedule(ddim_num_steps=S)
        k0, x_start = self.init_run(shape, x_init, strength, seed)
        if x_start is not None:
            input["x"] = x_start
        return self.plms_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, k0=k0)

    @torch.no_grad()
    def plms_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, k0=0):
        """plms.py:72-113, from step k0 (image-to-image) on."""
        b = shape[0]
        if input["x"] is None:
            input["x"] = torch.randn(shape, device=self.device)
        time_range = np.flip(self.ddim_timesteps)
        total_steps = self.ddim_timesteps.shape[0]
        alphas = self.alpha_generator_func(len(time_range)) if self.alpha_generator_func is not None else None
        tr = Trajectory(input)
        for i in range(k0, len(time_range)):
            if alphas is not None:
                self._set_alpha(alphas[i])
            ts, ts_next = self._timesteps(b, i, time_range)
            if mask is not None:  # inpainting blend (plms.py:99-103); host-level glue, unused by inference.py
                assert x0 is not None
                img_orig = self.diffusion.q_sample(x0, ts)
                input["x"] = img_orig * mask + (1. - mask) * input["x"]
            self._step([tr], ts, ts_next, total_steps - i - 1, uc, guidance_scale)
        return input["x"]
