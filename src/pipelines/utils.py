"""reference: src/pipelines/utils.py — the latent-interpolation method registry the pipeline file imports
(pipeline_pose2vid_long_edit_bkfill_roiclip.py:27, :327). It lives in mimo_b200/host/interpolation.py, where the
engine's sampler reads it for interpolation_factor >= 2; this module re-exports it so that the reference's unmodified
pipeline file and run scripts register the method the same way."""
from mimo_b200.host.interpolation import (  # noqa: F401
    get_tensor_interpolation_method,
    linear,
    set_tensor_interpolation_method,
    slerp,
)
