"""Write a self-supervised Human3.6M annotation file (train-ss.pkl) from a pretrained network:
lib.utils.prep_h36m.save_triangulations (the reference's unimplemented prep_h36m.py:211-213).

    python tools/prep_ss.py --cfg experiments/h36m/train-ss.yaml --model CKPT --root H36M_ROOT \
        --src annot/valid.pkl --dst annot/my-train-ss.pkl [--method robust|iterative|polynomial] \
        [--flip-test] [--threshold-px 15] [--batch 32] [--workers 8]

The model is built by get_pose_net from the config (MODEL.NUM_JOINTS decides the written layout:
16 from a 17-joint source is written in MPII order) and runs on the split-fp16 engine; CKPT holds
a state_dict, or a checkpoint dict with one under 'state_dict' ('module.' prefixes are removed).
--src / --dst are relative to --root unless absolute.  Prints the report as one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "epipolarpose_b200"))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--cfg", required=True)
    ap.add_argument("--model", required=True, help="checkpoint of the pretrained network")
    ap.add_argument("--root", required=True, help="Human3.6M root (images/ and annot/)")
    ap.add_argument("--src", required=True, help="dict-form annotation pickle to label")
    ap.add_argument("--dst", required=True, help="annotation pickle to write")
    ap.add_argument("--method", default="robust", choices=["robust", "iterative", "polynomial"])
    ap.add_argument("--flip-test", action="store_true")
    ap.add_argument("--threshold-px", type=float, default=15.0)
    ap.add_argument("--batch", type=int, default=32, help="frames (view tuples) per batch")
    ap.add_argument("--workers", type=int, default=8)
    a = ap.parse_args(argv)

    import torch
    import lib.dataset as dataset
    import lib.models as models
    from lib.core.config import config, update_config
    from lib.utils.prep_h36m import save_triangulations
    from epipolarpose_b200 import ops
    ops.device_check()
    update_config(a.cfg)
    config.MODEL.PRECISION = "f16x3"          # the predictors run the split-fp16 engine
    config.DATASET.ROOT = a.root
    model = models.pose3d_resnet.get_pose_net(config, is_train=False)
    ck = torch.load(a.model, map_location="cpu", weights_only=False)
    sd = ck.get("state_dict", ck) if isinstance(ck, dict) else ck
    sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
    model.load_state_dict(sd)
    model = model.cuda().eval()
    path = lambda p: p if os.path.isabs(p) else os.path.join(a.root, p)
    # the dataset supplies the crop geometry and the read path; its own db is the source when
    # the source lies in <root>/annot (read once more by the builder), else the test set
    src_dir, src_name = os.path.split(os.path.abspath(path(a.src)))
    in_annot = src_dir == os.path.abspath(os.path.join(a.root, "annot")) and src_name.endswith(".pkl")
    ds = dataset.h36m(config, a.root, src_name[:-4] if in_annot else config.DATASET.TEST_SET, False)
    report = save_triangulations(model, ds, path(a.src), path(a.dst), method=a.method, flip_test=a.flip_test,
                                 threshold_px=a.threshold_px, tuples_per_batch=a.batch, workers=a.workers)
    print(json.dumps(report))
    return report


if __name__ == "__main__":
    main()
