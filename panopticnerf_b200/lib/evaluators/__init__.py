"""The reference's ``lib.evaluators`` plugin surface: make_evaluator(cfg) -> Evaluator (evaluate / summarize / reset),
over the CUDA metric kernels of libpnr (pnr_eval_*)."""
from .make_evaluator import make_evaluator
from .panopticnerf import Evaluator, summarize_counts

__all__ = ["make_evaluator", "Evaluator", "summarize_counts"]
