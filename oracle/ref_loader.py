"""Load the UNMODIFIED reference module by path (test infrastructure only).

TEST INFRASTRUCTURE -- only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
import anything under oracle/.  This file is usable only where a checkout of the reference exists and
PWW_REFERENCE_ROOT names it; nothing else in the project needs it.  It is how the restatement in `pww_oracle.py` is pinned:
`tests/golden/make_golden.py` runs the real reference functions through this loader and commits their
outputs as fixtures.

The reference cannot be imported as a package here (SURVEY.md section 8c): `diffusers` is absent and
transformers>=5 has no `CLIPFeatureExtractor`.  Recipe: register placeholder `diffusers` modules, alias
`CLIPFeatureExtractor`, then exec `paint_with_words/paint_with_words.py` by path.  No reference source
is copied; nothing is written under the reference checkout.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("PWW_REFERENCE_ROOT", "")
_REF_FILE = os.path.join(REFERENCE_ROOT, "paint_with_words", "paint_with_words.py") if REFERENCE_ROOT else ""
_CACHE = {}


def reference_available() -> bool:
    return bool(_REF_FILE) and os.path.isfile(_REF_FILE)


def _install_stubs() -> None:
    if "diffusers" not in sys.modules:
        names = ("AutoencoderKL", "LMSDiscreteScheduler", "UNet2DConditionModel",
                 "StableDiffusionPipeline", "PNDMScheduler")
        root = types.ModuleType("diffusers")
        for n in names:
            setattr(root, n, type(n, (), {}))
        pipelines = types.ModuleType("diffusers.pipelines")
        sd = types.ModuleType("diffusers.pipelines.stable_diffusion")
        psd = types.ModuleType("diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion")
        psd.StableDiffusionPipelineOutput = type("StableDiffusionPipelineOutput", (), {})
        root.pipelines, pipelines.stable_diffusion, sd.pipeline_stable_diffusion = pipelines, sd, psd
        sys.modules.update({
            "diffusers": root,
            "diffusers.pipelines": pipelines,
            "diffusers.pipelines.stable_diffusion": sd,
            "diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion": psd,
        })
    # transformers is lazy: force the real module in first, then alias the removed name.
    from transformers import CLIPImageProcessor, CLIPTextModel, CLIPTokenizer  # noqa: F401
    tr = sys.modules["transformers"]
    if not hasattr(tr, "CLIPFeatureExtractor"):
        setattr(tr, "CLIPFeatureExtractor", CLIPImageProcessor)


def load_reference():
    """Return the reference `paint_with_words.py` as a module object (cached)."""
    if "mod" in _CACHE:
        return _CACHE["mod"]
    if not reference_available():
        raise FileNotFoundError(f"reference not present at {_REF_FILE}")
    _install_stubs()
    spec = importlib.util.spec_from_file_location("_pww_reference", _REF_FILE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _CACHE["mod"] = mod
    return mod
