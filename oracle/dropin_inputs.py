"""The inputs tests/test_dropin_cpu.py and oracle/gen_dropin_golden.py share: one synthetic clip for the
scene-compositing check, the tensors of the pipeline-utils check, and the digest the fixture stores per composited
frame. Test infrastructure, not product code."""
import hashlib

import numpy as np
import torch


def composite_inputs() -> dict:
    """A 7-frame 96x72 clip in two overlapping context windows (frames 3, 4 are composited twice: cross-fade) whose
    boxes touch different borders (different feather masks)."""
    from PIL import Image
    rng = np.random.RandomState(3)
    W, H, n_frames, overlay = 96, 72, 7, 2
    contexts = [[0, 1, 2, 3, 4], [3, 4, 5, 6]]
    bboxes = [(0, 60, 4, 72), (20, 96, 0, 50)]
    bk = [Image.fromarray(rng.randint(0, 256, (H, W, 3), dtype=np.uint8)) for _ in range(n_frames)]
    vid = [Image.fromarray(rng.randint(0, 256, (H, W, 3), dtype=np.uint8)) for _ in range(n_frames)]
    occ = [Image.fromarray(np.repeat(rng.randint(0, 256, (H, W, 1), dtype=np.uint8), 3, axis=2)) for _ in range(n_frames)]
    mask_list = [rng.rand(64, 64).astype(np.float32) for _ in range(16)]
    pads, padvs = [], []
    for k, ctx in enumerate(contexts):
        w_min, w_max, h_min, h_max = bboxes[k]
        bw, bh = w_max - w_min, h_max - h_min
        side = max(bw, bh)
        side += (16 - side % 16) % 16
        top = (side - bh) // 2
        left = (side - bw) // 2
        for _ in ctx:
            pads.append([side, side])
            padvs.append([top, side - bh - top, left, side - bw - left])
    video = torch.rand(3, sum(len(c) for c in contexts), 64, 64, generator=torch.Generator().manual_seed(3))
    return dict(n_frames=n_frames, overlay=overlay, contexts=contexts, bboxes=bboxes, bk=bk, vid=vid, occ=occ,
                mask_list=mask_list, pads=pads, padvs=padvs, video=video)


def utils_inputs():
    g = torch.Generator().manual_seed(3)
    a, b = torch.randn(4, 8, 8, generator=g), torch.randn(4, 8, 8, generator=g)
    return a, b, (0.0, 0.25, 0.5, 0.9)


def frame_digest(frame: np.ndarray) -> str:
    """SHA-256 of a composited frame (uint8 HxWx3): the fixture stores these instead of the frames themselves."""
    return hashlib.sha256(np.ascontiguousarray(frame, dtype=np.uint8).tobytes() + str(frame.shape).encode()).hexdigest()
