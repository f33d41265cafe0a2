"""PLMSSampler -- drop-in for ldm/models/diffusion/plms.py (same constructor and `sample`, both of `PLMSBase`)."""
from ._plms_common import PLMSBase


class PLMSSampler(PLMSBase):
    def plms_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, k0=0):
        """plms.py:72-113, from step k0 on: `PLMSBase.sample_loop`."""
        return self.sample_loop(shape, input, uc, guidance_scale, mask=mask, x0=x0, k0=k0)
