"""Drop-in for the reference's per-frame detection evaluation (opencood/utils/eval_utils.py:40-92 caluclate_tp_fp), which
opencood/tools/inference.py:171-185, inference_w_noise.py:160-170 and inference_heter_in_order.py:248-258 call after post_process
for IoU 0.3, 0.5 and 0.7.  With the boxes on the GPU the matching runs in heal_eval_tp_fp (csrc/eval.cu) and one device-to-host
copy brings back the flags, the sorted scores and the status; `result_stat` is extended exactly as the reference extends it, by
append_frame / append_packed, which the captured scene pipelines (heal_b200.graph) also use for their `result_stat`.
calculate_ap, voc_ap and eval_final_results (once per run, on the host) stay the reference's and read the same lists.

Where the result can differ from the reference's: the order of tied scores (the reference's np.argsort(-score) is not stable;
here ties go by ascending detection index), and the threshold test follows NumPy 2 (an fp32 IoU equal to float32(thr) is a TP).
Installed by heal_b200.install.install_gpu_eval()."""
import importlib

import torch

_BUFFERS = {}


def _gpu_boxes(t, n=None) -> bool:
    return (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 3
            and tuple(t.shape[1:]) == (8, 3) and (n is None or t.shape[0] == n))


def _reference():
    ref = caluclate_tp_fp.reference
    if ref is None:            # not installed: the reference module still holds its own function
        ref = importlib.import_module("opencood.utils.eval_utils").caluclate_tp_fp
    return ref


def caluclate_tp_fp(det_boxes, det_score, gt_boxes, result_stat, iou_thresh):
    """eval_utils.caluclate_tp_fp with the same name, arguments and effect on result_stat[iou_thresh]: 'tp' and 'fp' grow by one
    int per detection in descending score order, 'score' by the sorted scores (only when det_boxes is not None), 'gt' by G.
    CUDA fp32 (K, 8, 3) / (K,) / (G, 8, 3) inputs run on the GPU; anything else (CPU tensors, (N, 4, 2) boxes, other dtypes,
    det_boxes None) goes to the reference function.  A union of area 0 raises ZeroDivisionError, as the reference does."""
    if not (_gpu_boxes(det_boxes) and _gpu_boxes(gt_boxes) and isinstance(det_score, torch.Tensor) and det_score.is_cuda
            and det_score.dtype == torch.float32 and tuple(det_score.shape) == (det_boxes.shape[0],)
            and det_score.device == det_boxes.device == gt_boxes.device):
        return _reference()(det_boxes, det_score, gt_boxes, result_stat, iou_thresh)
    from .. import ops
    key = det_boxes.device
    buf = ops.eval_tp_fp(det_boxes.contiguous(), det_score.contiguous(), gt_boxes.contiguous(), [iou_thresh], _BUFFERS.get(key))
    _BUFFERS[key] = buf
    append_packed(result_stat, [iou_thresh], buf.packed.cpu(), det_boxes.shape[0], det_boxes.shape[0], gt_boxes.shape[0])


HEAL_EVAL_ZERO_UNION, HEAL_EVAL_OVER_CAPACITY = 1, 2       # status bits of include/heal_b200.h


def append_frame(result_stat, iou_thresh, scores, tp, n_gt: int):
    """Extend result_stat[iou_thresh] by one frame as the reference's caluclate_tp_fp does: 'score' by the frame's scores in
    descending order, 'fp' and 'tp' by one int per detection in that order, 'gt' by the frame's GT count.  `scores` (K,) fp32 and
    `tp` (K,) 0 / 1 are host tensors or arrays; K = 0 adds 'gt' only, as the reference does for det_boxes None."""
    stat = result_stat[iou_thresh]
    tp = [int(v) for v in tp.tolist()]
    stat['score'] += scores.tolist()
    stat['fp'] += [1 - v for v in tp]
    stat['tp'] += tp
    stat['gt'] += int(n_gt)


def append_packed(result_stat, thresholds, packed, K: int, K_cap: int, n_gt: int):
    """Append one frame to result_stat at each of `thresholds` from a host copy of EvalBuffers.packed: the status word, K_cap
    sorted scores and (len(thresholds), K_cap) flags, of which the first K are the frame's.  Raises before appending anything:
    ZeroDivisionError for a union of area 0 (where the reference raises it), RuntimeError for a count above the capacity."""
    from ..ops import EvalBuffers
    status, scores, tp = EvalBuffers.unpack(packed, K_cap, len(thresholds))
    if status & HEAL_EVAL_OVER_CAPACITY:
        raise RuntimeError(f"evaluation: a count above the capacity ({K_cap} detections); no flags were computed")
    if status & HEAL_EVAL_ZERO_UNION:
        raise ZeroDivisionError("float division by zero")
    for t, thr in enumerate(thresholds):
        append_frame(result_stat, thr, scores[:K], tp[t, :K], n_gt)


caluclate_tp_fp.reference = None
