"""The refinement unit (paper Sec. 3.3, the reference's refiner/) applied to the network's H36M poses.

The refiner's data are defined here as the H36M evaluation's `pred_to_save` (lib/dataset/h36m.py:346-348
of the reference): input = the root-relative camera-frame prediction `pred` in MPII order, target = the
matching `gt`, both [S, 16, 3] mm, float32 as the refiner reads them.  The reference never released the
script that wrote its refiner files, so this convention is inferred from its code.

  h36m_refined(poses, refiner_path, norm_path)  -> the four `Refined-*` entries of H36M_Integral.evaluate
  export_refiner_pairs(preds_in_img, dataset, path)  writes {'inp': pred, 'out': gt} for refiner/data.py
  load_refiner(refiner_path, norm_path)  the Refiner of a reference checkpoint, once per process"""
import pickle

import numpy as np
import torch

REFINED_NAMES = ('Refined-hm36_17j', 'Refined-hm36_17j_align', 'Refined-hm36_17j_14', 'Refined-hm36_17j_14_al')
HIP = 6
_REFINERS = {}


def load_refiner(refiner_path, norm_path):
    """refiner.model.Refiner of the checkpoint {'state_dict': ...} (the reference's layout, read as
    refiner/main.py's _restore reads it) with the four norm.pkl arrays; cached per process."""
    key = (refiner_path, norm_path)
    if key not in _REFINERS:
        from refiner.model import LinearModelPG, Refiner
        ckpt = torch.load(refiner_path, map_location="cpu", weights_only=False)
        sd = ckpt["state_dict"]
        L, n_in = sd["w1.weight"].shape
        model = LinearModelPG(linear_size=L, input_size=n_in, output_size=sd["w4.weight"].shape[0])
        model.load_state_dict(sd)
        with open(norm_path, "rb") as f:
            norm = pickle.load(f)
        _REFINERS[key] = Refiner(model.cuda().eval(), norm)
    return _REFINERS[key]


def check_refiner_config(test, mpii_order, num_joints):
    """(refiner_path, norm_path) of TEST.REFINER / TEST.REFINER_NORM, or None when REFINER is empty."""
    path = getattr(test, 'REFINER', '') if test is not None else ''
    if not path:
        return None
    norm = getattr(test, 'REFINER_NORM', '')
    if not norm:
        raise ValueError("TEST.REFINER needs TEST.REFINER_NORM (the refiner's norm.pkl)")
    if not mpii_order or num_joints != 16:
        raise ValueError("TEST.REFINER refines 16-joint poses in MPII order (DATASET.MPII_ORDER: true), got "
                         "%d joints%s" % (num_joints, "" if mpii_order else " in H36M order"))
    return path, norm


def pairs_of(poses):
    """poses [S, 16, 9] (epb_h36m_eval: pred | align_pred | gt) -> (pred, gt) float32 [S, 16, 3]."""
    return np.ascontiguousarray(poses[:, :, 0:3], np.float32), np.ascontiguousarray(poses[:, :, 6:9], np.float32)


def h36m_refined(poses, refiner_path, norm_path):
    """Refine the `pred` column and score it against `gt` with the hip dropped, as the refiner's
    evaluate does (epb_pose_errors) -> [(name, value)] * 4."""
    from refiner import data as rdata
    pred, gt = pairs_of(poses)
    if len(pred) == 0:
        return [(n, 0.0) for n in REFINED_NAMES]
    refined = load_refiner(refiner_path, norm_path).refine(pred)
    keep = [j for j in range(16) if j != HIP]
    metrics, _ = rdata.pose_errors(refined[:, keep], gt[:, keep])
    return list(zip(REFINED_NAMES, [float(v) for v in metrics.mean(axis=0)[:4]]))


def export_refiner_pairs(preds_in_img, dataset, path):
    """Write the refiner's training / validation file from image-space predictions of an H36M
    dataset in MPII order: {'inp': pred, 'out': gt}, float32 [S, 16, 3] (pickle).  Over `train-ss`,
    whose joints_3d are the triangulated pseudo-labels, these are the self-supervised pairs the
    refiner trains on; over `valid`, its validation file.  Returns the number of pairs."""
    from ..dataset.h36m_eval import evaluate_h36m
    preds = np.asarray(preds_in_img)[:, :, 0:3]
    S = preds.shape[0]
    if not bool(dataset.cfg.DATASET.MPII_ORDER) or preds.shape[1] != 16:
        raise ValueError("refiner pairs are 16-joint poses in MPII order (DATASET.MPII_ORDER: true)")
    gts = dataset.db[:S]
    get = lambda k: np.stack([np.asarray(g[k], dtype=np.float64).reshape(-1) for g in gts])
    gt = np.stack([np.asarray(g['joints_3d'], dtype=np.float64) for g in gts])
    _, _, details = evaluate_h36m(preds, gt, get('pelvis'), get('fl'), get('c_p'), mpii_order=True,
                                  return_poses=True)
    inp, out = pairs_of(details['poses'])
    with open(path, 'wb') as f:
        pickle.dump({'inp': inp, 'out': out}, f, protocol=4)
    return S
