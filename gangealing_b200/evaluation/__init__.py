"""Evaluation of a trained STN: PCK-Transfer (reference applications/pck.py), the test-time flip decision
(applications/__init__.py) and flow-smoothness scores (applications/flow_scores.py)."""
from .flips import determine_flips
from .flow_scores import filter_dataset, flow_scores, get_high_score_indices
from .pck import pck_transfer, pck_transfer_batch

__all__ = ["determine_flips", "filter_dataset", "flow_scores", "get_high_score_indices", "pck_transfer",
           "pck_transfer_batch"]
