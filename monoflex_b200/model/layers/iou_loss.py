"""`get_iou_3d` with the reference's module path and signature (model/layers/iou_loss.py:99-136), on the CUDA op
`mf_iou3d_corners` (csrc/mf_iou3d.cu, one thread per box pair). The reference clips the two bird's-eye-view rings with shapely
in a Python loop; here the clip is float64 on the GPU and the rest follows the reference's float32 steps. A ring is valid when
its four turns are non-zero with one sign; a simple but non-convex ring, which shapely accepts, is invalid here (DESIGN.md §9).
encode_box3d never builds one. There is no CPU path."""
import torch

from ..._lib import call


def get_iou_3d(pred_corners, target_corners):
    """pred_corners, target_corners: [N, 8, 3] float32 CUDA tensors in Anno_Encoder.encode_box3d's corner order.
    Returns the [N] float32 3D IoU of each pair on the same device; NaN corners give NaN."""
    for name, t in (("pred_corners", pred_corners), ("target_corners", target_corners)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("get_iou_3d: %s must be a torch.Tensor, got %s" % (name, type(t).__name__))
        if not t.is_cuda:
            raise RuntimeError("get_iou_3d: %s is on %s; monoflex_b200 runs on sm_90a GPUs only, no CPU fallback"
                               % (name, t.device))
        if t.dtype != torch.float32:
            raise TypeError("get_iou_3d: %s must be float32, got %s" % (name, t.dtype))
        if t.dim() != 3 or tuple(t.shape[1:]) != (8, 3):
            raise ValueError("get_iou_3d: %s must be [N, 8, 3], got %s" % (name, tuple(t.shape)))
    if pred_corners.shape[0] != target_corners.shape[0]:
        raise ValueError("get_iou_3d: %d predicted boxes vs %d target boxes" % (pred_corners.shape[0], target_corners.shape[0]))
    if pred_corners.device != target_corners.device:
        raise ValueError("get_iou_3d: inputs on %s and %s" % (pred_corners.device, target_corners.device))
    a, b = pred_corners.contiguous(), target_corners.contiguous()
    n = a.shape[0]
    out = torch.empty(n, dtype=torch.float32, device=a.device)
    if n:
        with torch.cuda.device(a.device):
            call("mf_iou3d_corners", a.data_ptr(), b.data_ptr(), n, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return out
