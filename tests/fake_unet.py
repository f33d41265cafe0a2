"""A fake UNet for the CPU tests of the request schedulers (`sample_requests`, `SamplingEngine`): its eps is a function
of each image's inputs, fuser scale and first conv, and it logs every forward.  The two sampler kernels are restated in
torch (`_plms_update`, `_latent_mean`), and `_alone` runs a request through its own sampler on a fresh fake, which is
what each scheduler's latent is compared with."""
import os
import sys
from dataclasses import replace
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from instancediffusion_b200.ldm.models.diffusion.batched import Request  # noqa: E402
from instancediffusion_b200.ldm.modules.attention import GatedSelfAttentionDense  # noqa: E402
from instancediffusion_b200.utils.model import alpha_generator, set_alpha_scale  # noqa: E402


def _plms_update(x, e_c, e_u, gs, olds, coefs, a_t, a_prev, s1m, e_out, x_out):
    e = e_c if e_u is None else e_u + gs * (e_c - e_u)
    ep = coefs[0] * e + sum(c * o for c, o in zip(coefs[1:], olds))
    xp = a_prev ** 0.5 * (x - s1m * ep) / a_t ** 0.5 + (1 - a_prev) ** 0.5 * ep
    if e_out is not None:
        e_out.copy_(e)
    x_out.copy_(xp)


def _latent_mean(xs, out):
    return out.copy_(torch.stack(xs).mean(0))


class FakeUNet(torch.nn.Module):
    """eps depends on the latent, the timestep, the context, the fuser scale and the first conv of each image.  Two tiny
    gated fusers carry the model's fuser scale (`scale` at construction), as `set_alpha_scale` sets it."""

    def __init__(self, scale=0.0):
        super().__init__()
        self.fusers = torch.nn.ModuleList([GatedSelfAttentionDense(8, 8, 1, 8) for _ in range(2)])
        set_alpha_scale(self, scale)
        self._first_conv_restored = False
        self._graphs, self._cat_cache = {}, {}
        self.calls, self.dropped = [], []

    def restore_first_conv_from_SD(self):
        self._first_conv_restored = True

    def forward_batched(self, inputs, *, scales=None, restored=None, per_image_conv=False):
        n = len(inputs)
        scales = [float(self.fusers[0].scale)] * n if scales is None else scales
        restored = [self._first_conv_restored] * n if restored is None else restored
        self.calls.append(dict(sizes=[i["x"].shape[0] for i in inputs], hw=[tuple(i["x"].shape[2:]) for i in inputs],
                               t=[int(i["timesteps"].reshape(-1)[0]) for i in inputs], scales=list(scales),
                               restored=list(restored), zero=[bool((i["x"] == 0).all()) for i in inputs]))
        return [0.1 * i["x"] + 1e-4 * i["timesteps"].float().view(-1, 1, 1, 1) + 0.01 * i["context"].mean()
                + 0.02 * s + 0.03 * float(r) for i, s, r in zip(inputs, scales, restored)]

    def drop_hoisted(self, inputs, keep=()):
        self.dropped.append(([id(i["context"]) for i in inputs], [id(i["context"]) for i in keep]))

    def trim_concats(self, keep):
        pass

    def trim_hoisted(self):
        pass


AGEN = partial(alpha_generator, type=[0.8, 0.0, 0.2])


def _req(seed, S, n=0, mis=0.0, size=64, ctx=77, alpha=AGEN, **kw):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((1, 4, size, size), generator=g)

    def inp():
        return dict(x=x, timesteps=None, context=torch.randn((1, ctx, 8), generator=g))
    ins = [inp() for _ in range(n + 1)] if n else inp()
    return Request(input=ins, uc=torch.zeros((1, ctx, 8)), guidance_scale=7.5, alpha_generator_func=alpha, mis=mis, S=S,
                   **kw)


def _fresh(req):
    if isinstance(req.input, list):
        x = req.input[0]["x"].clone()
        return replace(req, input=[dict(i, x=x) for i in req.input])
    return replace(req, input=dict(req.input, x=req.input["x"].clone()))


def _alone(diffusion, req, scale=0.0):
    """The request's latent from its own sampler on a fresh fake whose fusers are at `scale`."""
    from instancediffusion_b200.ldm.models.diffusion.plms import PLMSSampler
    from instancediffusion_b200.ldm.models.diffusion.plms_instance import PLMSSamplerInst
    model = FakeUNet(scale)
    req = _fresh(req)
    kw = dict(alpha_generator_func=req.alpha_generator_func, set_alpha_scale=set_alpha_scale)
    if isinstance(req.input, list):
        s = PLMSSamplerInst(diffusion, model, mis=req.mis, **kw)
    else:
        s = PLMSSampler(diffusion, model, **kw)
    return s.sample(S=req.S, shape=(1, 4) + tuple(req.input[0]["x"].shape[2:] if isinstance(req.input, list)
                                                 else req.input["x"].shape[2:]), input=req.input, uc=req.uc,
                    guidance_scale=req.guidance_scale)
