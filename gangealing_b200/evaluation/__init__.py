"""Evaluation of a trained STN: PCK-Transfer (reference applications/pck.py), the test-time flip decision
(applications/__init__.py), flow-smoothness scores (applications/flow_scores.py) and the congealing visualisations
(applications/vis_correspondence.py, propagate_to_images.py) and dataset congealing (applications/congeal_dataset.py)."""
from .congeal import congeal_dataset, congeal_images
from .flips import determine_flips
from .flow_scores import filter_dataset, flow_scores, get_high_score_indices
from .pck import pck_transfer, pck_transfer_batch
from .propagate import average_png, load_dense_label, propagate_to_images, save_propagation
from .visuals import (average_congealed_image, congealing_average_frames, label_propagation_frames, labeled_average_frames,
                      smooth_congealing, smooth_correspondence)

__all__ = ["average_congealed_image", "average_png", "congeal_dataset", "congeal_images", "congealing_average_frames",
           "determine_flips", "filter_dataset",
           "flow_scores", "get_high_score_indices", "label_propagation_frames", "labeled_average_frames",
           "load_dense_label", "pck_transfer", "pck_transfer_batch", "propagate_to_images", "save_propagation",
           "smooth_congealing", "smooth_correspondence"]
