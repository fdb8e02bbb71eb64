"""TEST INFRASTRUCTURE (never imported by mimo_b200/): numpy restatement of run_edit.py's per-frame scene compositing
(the original project's run_edit.py:282-300) — the blend chain after the generated frame has been resized, un-padded and pasted
on the white canvas. The loop lives inside MIMO.run, behind TensorFlow / model loading at import time, so it cannot be
imported; it is restated line by line, with numpy's own type promotion doing the arithmetic, and PINNED against the
reference's own statements: tests/test_dropin_cpu.py extracts the loop from run_edit.py by AST, executes it with
tools/util.py's get_mask on a synthetic clip and requires byte-identical frames from host/composite.py + this oracle:

    res_image = res_image * mask_full[:, :, np.newaxis] + bk_image * (1 - mask_full[:, :, np.newaxis])      :284
    occ_mask = occ_mask / 255.0;  res_image = res_image * (1 - occ) + vid_image * occ                       :288-292
    res_images[i] = res_images[i] * (1 - factor) + res_image * factor   (overlapping clips)                 :296-297
    res_images[i] = res_images[i].astype(np.uint8)                                                          :298
"""
import numpy as np


def composite_frame(canvas: np.ndarray, bk: np.ndarray, mask_full: np.ndarray, occ=None, vid=None, prev=None,
                    factor: float = 0.0) -> np.ndarray:
    """canvas / bk / vid / prev: uint8 [H, W, 3]; mask_full: float32 [H, W]; occ: uint8 [H, W] (channel 0 of the
    occlusion mask image); factor: (i - start_i + 1) / (overlay + 1), a Python float."""
    assert canvas.dtype == np.uint8 and bk.dtype == np.uint8 and mask_full.dtype == np.float32
    res_image = canvas * mask_full[:, :, np.newaxis] + bk * (1 - mask_full[:, :, np.newaxis])
    if occ is not None:
        occ_mask = occ.astype(np.uint8) / 255.0
        res_image = res_image * (1 - occ_mask[:, :, np.newaxis]) + vid * occ_mask[:, :, np.newaxis]
    if prev is None:
        out = res_image
    else:
        out = prev * (1 - factor) + res_image * factor
    return out.astype(np.uint8)
