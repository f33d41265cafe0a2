"""PLMSSampler -- drop-in for ldm/models/diffusion/plms.py (same constructor and `sample`)."""
import torch

from ._plms_common import PLMSBase


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
        return self.sample_loop(shape, input, uc, guidance_scale, mask=mask, x0=x0, k0=k0)
