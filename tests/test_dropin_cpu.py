"""Drop-in boundary proof (SURVEY.md §8b) on CPU, against data the original project's own files produced
(tests/golden/dropin_reference.npz; oracle/gen_dropin_golden.py regenerates it from a checkout of that project):
the scene-compositing helper against the frames run_edit.py's post-processing loop produced on the same synthetic clip,
and the overlay's src/pipelines/utils.py against the reference file's linear / slerp results on the same inputs.
The shipped pipeline itself is pinned to the golden clip of the reference's pipeline in tests/test_pipeline_plumbing_cpu.py
and tests/test_engine_gpu.py."""
import numpy as np
import pytest
import torch

from oracle.dropin_inputs import composite_inputs, frame_digest, utils_inputs


@pytest.fixture(scope="module")
def dropin_golden(golden_dir):
    with np.load(golden_dir / "dropin_reference.npz") as z:
        return {k: z[k] for k in z.files}


def test_scene_compositing_matches_the_reference_loop(monkeypatch, dropin_golden):
    """run_edit.py's post-processing loop (:253-304) with tools/util.py's own get_mask - its frames on this synthetic clip
    are stored as digests in tests/golden/dropin_reference.npz - against mimo_b200.host.composite.composite_clip on the
    same clip (oracle/dropin_inputs.py). The blend kernel needs a GPU, so here (and only here) ops.composite_frame is the numpy oracle: this pins the helper's host logic (PIL resize / crop / paste,
    INTER_AREA mask resize, mask placement, cross-fade factor, 16-way mask choice) AND the oracle's arithmetic to the
    reference's code; the kernel is pinned to the oracle bit for bit on the GPU (tests/test_clip_composite_gpu.py)."""
    from mimo_b200 import ops
    from mimo_b200.host import composite
    from oracle.composite_oracle import composite_frame
    c = composite_inputs()
    n_frames = c["n_frames"]

    # ---- this repo's helper, with the blend evaluated by the oracle instead of the kernel ----
    def blend_on_cpu(canvas, bkf, mask, *, occ=None, vid=None, prev=None, factor=0.0, out=None):
        f = lambda t: None if t is None else t.cpu().numpy()
        return torch.from_numpy(composite_frame(f(canvas), f(bkf), f(mask), f(occ), f(vid), f(prev), factor))

    monkeypatch.setattr(ops, "composite_frame", blend_on_cpu)
    args = (c["contexts"], c["bboxes"], c["bk"], c["vid"])
    rest = (c["pads"], c["padvs"], c["mask_list"], n_frames, c["overlay"])
    got = composite.composite_clip(c["video"], *args, c["occ"], *rest, device="cpu")
    for i in range(n_frames):
        assert got[i] is not None
        assert frame_digest(np.asarray(got[i])) == dropin_golden["composite_occ"][i], i
    # and without an occlusion mask (animate-style templates, run_edit.py:262-265)
    got = composite.composite_clip(c["video"], *args, None, *rest, device="cpu")
    for i in range(n_frames):
        assert frame_digest(np.asarray(got[i])) == dropin_golden["composite_no_occ"][i], i


def test_overlay_pipeline_utils_equal_the_reference(dropin_golden):
    """src/pipelines/utils.py (imported by the reference's pipeline file, dead at interpolation_factor = 1): the overlay's
    linear and slerp against the reference file's results on the same inputs, bit for bit, and its registry."""
    import src.pipelines.utils as ours
    a, b, ts = utils_inputs()
    for i, t in enumerate(ts):
        assert torch.equal(ours.linear(a, b, t), torch.from_numpy(dropin_golden["linear"][i]))
        assert torch.equal(ours.slerp(a, b, t), torch.from_numpy(dropin_golden["slerp"][i]))
        # nearly parallel: the linear branch
        assert torch.equal(ours.slerp(a, a * 1.0001, t), torch.from_numpy(dropin_golden["slerp_parallel"][i]))
    for flag, name in ((True, "slerp"), (False, "linear")):
        ours.set_tensor_interpolation_method(flag)
        assert ours.get_tensor_interpolation_method().__name__ == name
