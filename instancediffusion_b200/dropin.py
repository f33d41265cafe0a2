"""Drop-in seam.  The reference has no FFI: its plug-in mechanism is YAML `target:` dotted paths
resolved by importlib (ldm/util.py:71-84; configs/test_*.yaml:2,9,27,43,64,76) plus a handful of
direct imports in inference.py:14-22.  `install()` makes exactly the hot-path *leaf modules* of
SURVEY.md section 8b resolve to this package's mirrors:

    ldm.util
    ldm.modules.attention
    ldm.modules.diffusionmodules.{openaimodel, text_grounding_net, util, convnext}
    ldm.models.diffusion.{plms, plms_instance, ldm, ddpm}
    grounding_input.text_grounding_tokinzer_input
    utils.model  (set_alpha_scale / alpha_generator only; everything else stays the reference's)
    ldm.models.autoencoder, ldm.modules.diffusionmodules.model   (first stage: AutoencoderKL.decode right
        after the sampler loop, inference.py:96; `install(first_stage=False)` leaves it to the reference)
    ldm.modules.encoders.modules   (only with `install(text_encoder=True)`: FrozenCLIPEmbedder, configs/*.yaml:72)

With a reference checkout on sys.path (or passed as `reference_root` / $IDIFF_REF) the *parent*
packages stay the reference's own (`ldm`, `ldm.modules`, `ldm.models`, `utils` are namespace
packages there), so every module that is not mirrored -- `ldm.modules.encoders.modules`, `utils.input`,
`utils.checkpoint`, `dataset.*` -- keeps importing from the reference's files, and a name a
mirrored module does not define (e.g. `ldm.modules.attention.LinearAttention`, imported by the
reference's VAE, diffusionmodules/model.py:9) is fetched lazily from the reference's own file of
that module.  Without a checkout (the GPU box, unit tests) the mirrors' packages stand in as
parents, which is enough for configs that name only hot-path targets.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types
from typing import Optional

_MAP = {
    "ldm.util": "instancediffusion_b200.ldm.util",
    "ldm.modules.attention": "instancediffusion_b200.ldm.modules.attention",
    "ldm.modules.diffusionmodules.openaimodel": "instancediffusion_b200.ldm.modules.diffusionmodules.openaimodel",
    "ldm.modules.diffusionmodules.text_grounding_net": "instancediffusion_b200.ldm.modules.diffusionmodules.text_grounding_net",
    "ldm.modules.diffusionmodules.util": "instancediffusion_b200.ldm.modules.diffusionmodules.util",
    "ldm.modules.diffusionmodules.convnext": "instancediffusion_b200.ldm.modules.diffusionmodules.convnext",
    "ldm.models.diffusion.plms": "instancediffusion_b200.ldm.models.diffusion.plms",
    "ldm.models.diffusion.plms_instance": "instancediffusion_b200.ldm.models.diffusion.plms_instance",
    "ldm.models.diffusion.ldm": "instancediffusion_b200.ldm.models.diffusion.ldm",
    "ldm.models.diffusion.ddpm": "instancediffusion_b200.ldm.models.diffusion.ddpm",
    "grounding_input.text_grounding_tokinzer_input": "instancediffusion_b200.grounding_input.text_grounding_tokinzer_input",
}
_FIRST_STAGE = {
    "ldm.models.autoencoder": "instancediffusion_b200.ldm.models.autoencoder",
    "ldm.modules.diffusionmodules.model": "instancediffusion_b200.ldm.modules.diffusionmodules.model",
}
# opt-in (install(text_encoder=True)): the CLIP text tower of FrozenCLIPEmbedder on the H100 kernels; the other
# encoder classes of that file (BERT, FrozenCLIPTextEmbedder, ...) are fetched lazily from the reference's own file
_TEXT_ENCODER = {
    "ldm.modules.encoders.modules": "instancediffusion_b200.ldm.modules.encoders.modules",
}
_PKGS = {
    "ldm": "instancediffusion_b200.ldm",
    "ldm.modules": "instancediffusion_b200.ldm.modules",
    "ldm.modules.diffusionmodules": "instancediffusion_b200.ldm.modules.diffusionmodules",
    "ldm.models": "instancediffusion_b200.ldm.models",
    "ldm.models.diffusion": "instancediffusion_b200.ldm.models.diffusion",
    "grounding_input": "instancediffusion_b200.grounding_input",
}
_installed: list = []
_REF_PREFIX = "_idiff_reference_original."


def find_reference_root(explicit: Optional[str] = None) -> Optional[str]:
    """The reference checkout: explicit argument, $IDIFF_REF, else the first sys.path entry (or the cwd,
    which is how `python inference.py` is run) that holds ldm/modules/attention.py."""
    cands = [explicit, os.environ.get("IDIFF_REF")] + list(sys.path) + [os.getcwd()]
    for c in cands:
        if c is None:
            continue
        c = c or os.getcwd()
        if os.path.isfile(os.path.join(c, "ldm", "modules", "attention.py")) and \
                os.path.isdir(os.path.join(c, "grounding_input")):
            return os.path.abspath(c)
    return None


def _reference_original(alias: str, root: str):
    """Load the reference's own file of a shadowed module under a private name (cached)."""
    name = _REF_PREFIX + alias
    mod = sys.modules.get(name)
    if mod is not None:
        return mod
    path = os.path.join(root, *alias.split(".")) + ".py"
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    try:
        spec.loader.exec_module(mod)
    except BaseException:
        sys.modules.pop(name, None)
        raise
    return mod


def _add_fallback(mirror: types.ModuleType, alias: str, root: str) -> None:
    """PEP 562 module __getattr__: names the mirror does not define come from the reference's file."""
    def __getattr__(attr, _alias=alias, _root=root):
        if attr.startswith("__"):
            raise AttributeError(attr)
        try:
            return getattr(_reference_original(_alias, _root), attr)
        except AttributeError:
            raise AttributeError(f"module '{_alias}' (instancediffusion_b200 mirror) has no attribute '{attr}', "
                                 f"and neither has the reference's {_alias}") from None
    mirror.__getattr__ = __getattr__


def _bind(alias: str, module: types.ModuleType) -> None:
    sys.modules[alias] = module
    _installed.append(alias)
    if "." in alias:
        parent, leaf = alias.rsplit(".", 1)
        if parent in sys.modules:
            setattr(sys.modules[parent], leaf, module)


def install(shadow_utils_model: bool = True, reference_root: Optional[str] = None,
            first_stage: bool = True, text_encoder: bool = False) -> Optional[str]:
    """Alias the mirror leaf modules under the reference's import paths; returns the reference root
    that keeps serving the non-mirrored modules (None if no checkout is visible)."""
    root = find_reference_root(reference_root)
    from .utils import model as um
    leaf_map = {**_MAP, **(_FIRST_STAGE if first_stage else {}), **(_TEXT_ENCODER if text_encoder else {})}
    if root is not None:
        if root not in sys.path:
            sys.path.insert(0, root)
        # parents: the reference's own (namespace) packages
        for pkg in _PKGS:
            for stale in [k for k in sys.modules if k == pkg]:
                m = sys.modules[stale]
                if getattr(m, "__name__", "").startswith("instancediffusion_b200"):
                    del sys.modules[stale]  # left over from a checkout-less install()
            importlib.import_module(pkg)
        for alias, real in leaf_map.items():
            mirror = importlib.import_module(real)
            if os.path.isfile(os.path.join(root, *alias.split(".")) + ".py"):
                _add_fallback(mirror, alias, root)
            _bind(alias, mirror)
        if shadow_utils_model:
            importlib.import_module("utils")
            try:
                real = importlib.import_module("utils.model")  # the reference's, with our classes already in place
                real.set_alpha_scale = um.set_alpha_scale
                real.alpha_generator = um.alpha_generator
            except ImportError as exc:
                # a dependency of the reference's utils/model.py (omegaconf, tensorboard, ...) is missing in this
                # environment: serve the two hot-path functions, report the real cause for anything else
                shim = types.ModuleType("utils.model")
                shim.set_alpha_scale = um.set_alpha_scale
                shim.alpha_generator = um.alpha_generator
                shim.__file__ = os.path.join(root, "utils", "model.py")
                cause = exc

                def __getattr__(attr, _cause=cause):
                    if attr.startswith("__"):
                        raise AttributeError(attr)
                    raise ImportError(f"utils.model.{attr} lives in the reference's utils/model.py, which failed "
                                      f"to import here: {_cause}", name=getattr(_cause, "name", None))
                shim.__getattr__ = __getattr__
                _bind("utils.model", shim)
        return root
    # no checkout: the mirrors' packages stand in as parents
    pkgs = dict(_PKGS)
    if text_encoder:
        pkgs["ldm.modules.encoders"] = "instancediffusion_b200.ldm.modules.encoders"
    for alias, real in {**pkgs, **leaf_map}.items():
        sys.modules[alias] = importlib.import_module(real)
        _installed.append(alias)
    if shadow_utils_model:
        pkg = sys.modules.get("utils")
        if pkg is None:
            pkg = types.ModuleType("utils")
            pkg.__path__ = []  # namespace-like
            sys.modules["utils"] = pkg
            _installed.append("utils")
        shim = types.ModuleType("utils.model")
        shim.set_alpha_scale = um.set_alpha_scale
        shim.alpha_generator = um.alpha_generator
        sys.modules["utils.model"] = shim
        _installed.append("utils.model")
        pkg.model = shim
    return None


def uninstall() -> None:
    for alias in _installed:
        sys.modules.pop(alias, None)
    _installed.clear()
    for k in [k for k in sys.modules if k.startswith(_REF_PREFIX)]:
        del sys.modules[k]
