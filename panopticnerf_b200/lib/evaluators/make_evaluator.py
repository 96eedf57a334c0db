"""make_evaluator(cfg) -> Evaluator   (the reference's lib/evaluators/make_evaluator.py, not in the mount): the class
`Evaluator` of cfg.evaluator_path (a file) when given, else of cfg.evaluator_module."""
from __future__ import annotations

import importlib
import importlib.util

DEFAULT_MODULE = "panopticnerf_b200.lib.evaluators.panopticnerf"


def make_evaluator(cfg):
    path = getattr(cfg, "evaluator_path", None)
    if path:
        spec = importlib.util.spec_from_file_location("pnr_evaluator_plugin", path)
        if spec is None or spec.loader is None:
            raise ImportError(f"make_evaluator: cannot load {path}")
        module = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(module)
    else:
        module = importlib.import_module(getattr(cfg, "evaluator_module", None) or DEFAULT_MODULE)
    return module.Evaluator(cfg)
