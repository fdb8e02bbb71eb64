"""Writes tests/golden/dropin_reference.npz: what the original MIMO project's own code computes on the inputs of
tests/test_dropin_cpu.py (oracle/dropin_inputs.py) - run_edit.py's post-processing loop (with tools/util.py's get_mask)
with and without an occlusion mask (a SHA-256 digest per frame), and src/pipelines/utils.py's linear / slerp.
Test infrastructure, not product code.

Usage:  MIMO_REFERENCE=<checkout of the original project> python oracle/gen_dropin_golden.py"""
import ast
import importlib.util
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path[:0] = [str(ROOT / "oracle" / "diffusers_shim"), str(ROOT / "tests" / "compat")]  # what the reference imports


from oracle.dropin_inputs import composite_inputs, frame_digest, utils_inputs  # noqa: E402


def _load(path: Path, name: str):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main(ref: Path) -> None:
    import cv2
    from PIL import Image
    out = {}

    # run_edit.py MIMO.run: the statements that set video_idx and res_images, and the loop over context_list
    c = composite_inputs()
    ref_util = _load(ref / "tools" / "util.py", "_reference_tools_util")
    tree = ast.parse((ref / "run_edit.py").read_text())
    run = next(f for cl in tree.body if isinstance(cl, ast.ClassDef) and cl.name == "MIMO"
               for f in cl.body if isinstance(f, ast.FunctionDef) and f.name == "run")
    loop = next(st for st in run.body if isinstance(st, ast.For) and isinstance(st.iter, ast.Call)
                and getattr(st.iter.func, "id", "") == "enumerate" and getattr(st.iter.args[0], "id", "") == "context_list")
    init = next(st for st in run.body if isinstance(st, ast.Assign) and getattr(st.targets[0], "id", "") == "res_images")
    idx0 = next(st for st in run.body if isinstance(st, ast.Assign) and getattr(st.targets[0], "id", "") == "video_idx")
    mod = ast.Module(body=[idx0, init, loop], type_ignores=[])
    ast.fix_missing_locations(mod)
    me = SimpleNamespace(args=SimpleNamespace(L=c["n_frames"]), mask_list=c["mask_list"])
    for key, occ in (("composite_occ", c["occ"]), ("composite_no_occ", None)):
        ns = dict(np=np, cv2=cv2, Image=Image, get_mask=ref_util.get_mask, self=me, context_list=c["contexts"],
                  bbox_clip_list=c["bboxes"], bk_images_ori=c["bk"], vid_images_ori=c["vid"], occ_mask_images=occ,
                  clip_pad_list_context=c["pads"], clip_padv_list_context=c["padvs"], video=c["video"],
                  overlay=c["overlay"])
        exec(compile(mod, "run_edit.py:MIMO.run[post-process]", "exec"), ns)
        out[key] = np.array([frame_digest(np.asarray(f)) for f in ns["res_images"]])

    utils = _load(ref / "src" / "pipelines" / "utils.py", "_reference_pipeline_utils")
    a, b, ts = utils_inputs()
    out["linear"] = np.stack([utils.linear(a, b, t).numpy() for t in ts])
    out["slerp"] = np.stack([utils.slerp(a, b, t).numpy() for t in ts])
    out["slerp_parallel"] = np.stack([utils.slerp(a, a * 1.0001, t).numpy() for t in ts])

    dst = ROOT / "tests" / "golden" / "dropin_reference.npz"
    np.savez_compressed(dst, **out)
    print(f"wrote {dst} ({dst.stat().st_size} bytes): {', '.join(f'{k} {v.shape} {v.dtype}' for k, v in out.items())}")


if __name__ == "__main__":
    if not os.environ.get("MIMO_REFERENCE"):
        raise SystemExit(__doc__)
    torch.set_num_threads(1)
    main(Path(os.environ["MIMO_REFERENCE"]))
