"""The latent-interpolation method registry of the reference's src/pipelines/utils.py, which its pipeline file imports
(pipeline_pose2vid_long_edit_bkfill_roiclip.py:27, :294-334, :566-567). `set_tensor_interpolation_method(is_slerp)`
chooses how Pose2VideoPipeline(interpolation_factor=k >= 2) fills the k-1 frames between each pair of denoised latent
frames. The sampler runs the registered method as the mimo_interpolate_frames kernel, so only the two functions below
can be registered; `linear` and `slerp` here are the tensor-level definitions (the overlay's src/pipelines/utils.py
re-exports this module)."""
import torch

_method = None


def get_tensor_interpolation_method():
    return _method


def set_tensor_interpolation_method(is_slerp):
    global _method
    _method = slerp if is_slerp else linear


def linear(v1, v2, t):
    return (1.0 - t) * v1 + t * v2  # this evaluation order: bit-identical to the reference's


def slerp(v0: torch.Tensor, v1: torch.Tensor, t: float, DOT_THRESHOLD: float = 0.9995) -> torch.Tensor:
    cos = (v0 / v0.norm() * (v1 / v1.norm())).sum()
    if cos.abs() > DOT_THRESHOLD:  # nearly parallel: the great-circle formula is ill-conditioned
        return (1.0 - t) * v0 + t * v1
    theta = cos.acos()
    return (torch.sin((1.0 - t) * theta) * v0 + torch.sin(t * theta) * v1) / torch.sin(theta)


def kernel_method(fn) -> int:
    """The mimo_interpolate_frames method of a registered function (by identity): 0 linear, 1 slerp."""
    if fn is None:
        raise TypeError("interpolation_factor >= 2 needs an interpolation method: call "
                        "set_tensor_interpolation_method(is_slerp) first (src/pipelines/utils.py)")
    if fn is linear:
        return 0
    if fn is slerp:
        return 1
    raise NotImplementedError(f"interpolation method {fn!r}: only the registry's linear and slerp run on the engine")
