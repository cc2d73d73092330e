"""Generate tests/golden/aliked/al_*.pt by running the UNMODIFIED reference ALIKED on the CPU.

    make -C oracle -f aliked_ref.mk         # copies the reference's lightglue/aliked.py to oracle/_ref/aliked_ref.py
    python oracle/make_golden_aliked.py [case ...]

The reference file is loaded by path with the stand-ins of oracle/aliked_ref_loader.py (a ``kornia.color`` stub that
must never be called -- the fixtures feed 3-channel images --, a minimal ``Extractor`` base, and a checkpoint download
that returns the seeded synthetic weights of oracle/aliked_synth.py).  Fixtures store the recipe, checksums of the
regenerated image / weights, the reference's state_dict key names and shapes, the integer NMS positions (the reference
DKD run with ``sub_pixel=False`` on the same score map) and the outputs.  Every case is checked to be well posed: no
NMS-surviving score within 1e-5 of the threshold, no NMS window whose two largest scores are within 1e-5, and, where
candidates are ranked, no two neighbours in the ranking within 1e-7.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lightglue_b200 import synth  # noqa: E402
from oracle import aliked_ref_loader as loader  # noqa: E402
from oracle import aliked_synth as als  # noqa: E402

# a directory of their own: the matcher suites take every tests/golden/*.pt that is not sp_*
OUT = os.path.join(ROOT, "tests", "golden", "aliked")
# CPU threads of the fixture run.  oneDNN splits a convolution's sums by thread count, so an fp32 result is reproducible
# to the last bits only with the same count: the oracle test runs with it too.
FIXTURE_THREADS = 8

CASES = {
    # default conf: threshold 0.2, n_limit 20000 (no limit reached), row-major order
    "al_240x320": dict(h=240, w=320, b=1, seed=1, model="aliked-n16", conf={}),
    # replicate padding to 224 x 320 is asymmetric on both axes (top 10 / bottom 11, left 1 / right 2)
    "al_odd_203x317": dict(h=203, w=317, b=1, seed=2, model="aliked-n16", conf={}),
    # threshold mode with max_num_keypoints below the candidate count: candidates sorted by score
    "al_thr_top300": dict(h=240, w=320, b=1, seed=3, model="aliked-n16", conf=dict(max_num_keypoints=300)),
    # top-k mode (detection_threshold <= 0, max_num_keypoints > 0), batch of two
    "al_topk_b2": dict(h=192, w=256, b=2, seed=4, model="aliked-n16", conf=dict(detection_threshold=-1, max_num_keypoints=400)),
    # per-image border from image_size (DKD.forward): image 0 declares 300 x 200 valid pixels of its 320 x 240.  The last
    # image declares its full size: DKD.forward's loop over image_size rebinds its `w, h`, which then decode the flat
    # indices and scale the keypoints of EVERY image, so only a full-size last image leaves positions intact (a
    # documented deviation of lightglue_b200.aliked, which keeps each image's own pixel positions)
    "al_b2_image_size": dict(h=240, w=320, b=2, seed=5, model="aliked-n16", conf=dict(max_num_keypoints=256),
                             image_size=[[300.0, 200.0], [320.0, 240.0]]),
    # narrow channels, dim 64
    "al_t16": dict(h=240, w=320, b=1, seed=6, model="aliked-t16", conf={}),
    # 32 SDDH sample positions
    "al_n32": dict(h=160, w=224, b=1, seed=7, model="aliked-n32", conf={}),
}


def _nms_positions(model, score_map, image_size):
    """Integer NMS positions (x, y), in output order: the reference's DKD without the soft-argmax."""
    kps, _, _ = model.dkd(score_map, sub_pixel=False, image_size=image_size)
    h, w = score_map.shape[-2:]
    wh = torch.tensor([w - 1, h - 1], dtype=torch.float32)
    return [torch.round((k + 1) / 2 * wh).long() for k in kps]


def _check_well_posed(model, score_map, nms, thr, ranked):
    r = model.conf.nms_radius
    pad = torch.nn.functional.pad(score_map, (r, r, r, r), value=-1.0)
    win = pad.unfold(2, 2 * r + 1, 1).unfold(3, 2 * r + 1, 1).reshape(*score_map.shape, -1)
    top2 = win.topk(2, dim=-1).values
    for b, pos in enumerate(nms):
        s = score_map[b, 0, pos[:, 1], pos[:, 0]]
        t2 = top2[b, 0, pos[:, 1], pos[:, 0]]
        assert float((t2[:, 0] - t2[:, 1]).min()) > 1e-5, "NMS near-tie"
        if thr > 0:
            assert float((s - thr).abs().min()) > 1e-5, "score within 1e-5 of the threshold"
        if ranked and len(s) > 1:
            ss = s.sort(descending=True).values
            assert float((ss[:-1] - ss[1:]).min()) > 1e-7, "near-tie in the ranking"


def _offset_stats(model, image):
    """Largest |offset| of the deformable convolutions and of SDDH (recorded: the fixtures must exercise them)."""
    stats = {}
    hooks = []
    for name in ("block3.conv1", "block3.conv2", "block4.conv1", "block4.conv2"):
        mod = model.get_submodule(name).offset_conv
        hooks.append(mod.register_forward_hook(lambda m, i, o, n=name: stats.__setitem__(n, float(o.abs().max()))))
    hooks.append(model.desc_head.offset_conv.register_forward_hook(
        lambda m, i, o: stats.__setitem__("sddh_abs_mean", float(o.abs().mean()))))
    model({"image": image})
    for h in hooks:
        h.remove()
    return stats


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(FIXTURE_THREADS)
    os.makedirs(OUT, exist_ok=True)
    only = set(sys.argv[1:])  # optional: names of the cases to (re)generate
    for name, rc in CASES.items():
        if only and name not in only:
            continue
        weights = als.make_aliked_state_dict(rc["model"], 0)
        model = loader.build_model(weights, model_name=rc["model"], **rc["conf"])
        conf = model.conf
        image_size = torch.tensor(rc["image_size"]) if "image_size" in rc else None
        rc = dict(rc, rejected_seeds=[])
        while True:  # a seed whose case is ill posed (see the module docstring) is replaced by seed + 100, and recorded
            image = als.make_image(rc["h"], rc["w"], rc["b"], rc["seed"])
            _, score_map = model.extract_dense_map(image)
            nms = _nms_positions(model, score_map, image_size)
            ranked = (conf.detection_threshold <= 0) or (
                conf.max_num_keypoints > 0 and nms[0].shape[0] >= conf.max_num_keypoints)
            try:
                _check_well_posed(model, score_map, nms, conf.detection_threshold, ranked)
                break
            except AssertionError as e:
                rc["rejected_seeds"].append((rc["seed"], str(e)))
                rc["seed"] += 100
        data = {"image": image} if image_size is None else {"image": image, "image_size": image_size}
        out = model(data)
        res = {k: [t.clone() for t in out[k]] for k in ("keypoints", "keypoint_scores", "descriptors")}
        res["nms_positions"] = nms
        # keep the fixtures small: above 600 keypoints only every 4th descriptor row is stored
        res["desc_stride"] = [4 if t.shape[0] > 600 else 1 for t in res["descriptors"]]
        res["descriptors"] = [t[::st].clone() for t, st in zip(res["descriptors"], res["desc_stride"])]
        fix = {
            "recipe": rc,
            "conf": {k: getattr(conf, k) for k in ("model_name", "max_num_keypoints", "detection_threshold", "nms_radius")},
            "image_checksum": synth.checksum(image),
            "weights_checksum": {k: synth.checksum(v) for k, v in weights.items() if v.dtype == torch.float32},
            "state_dict_layout": [(k, tuple(v.shape)) for k, v in model.state_dict().items()],
            "offset_stats": _offset_stats(model, image),
            "out": res,
        }
        torch.save(fix, os.path.join(OUT, name + ".pt"))
        print(name, [tuple(t.shape) for t in res["keypoints"]], fix["offset_stats"], rc["rejected_seeds"])


if __name__ == "__main__":
    main()
