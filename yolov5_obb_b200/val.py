"""Host-side mirror of the per-image metric block of the reference's validation loop (val.py:209-250 and
process_batch :69-92), executed for a whole batch by ONE kernel (csrc/val_match.cu, SURVEY section 8f rank 3)."""
import torch

from . import _lib


def match_batch(dets: torch.Tensor, counts: torch.Tensor, targets: torch.Tensor, shapes, iouv: torch.Tensor,
                want_geometry: bool = True):
    """dets [B, max_det, 7] + counts [>= B] int64: the packed pair non_max_suppression_obb(..., return_packed=True / "async")
    returns (rows (cx, cy, l, s, theta, conf, cls) in network-input pixels).
    targets [nt, >= 7]: (image, cls, cx, cy, l, s, theta, ...) as val.py:199 holds them (pixels).
    shapes: per image ((h_raw, w_raw), ((gain_h, gain_w), (pad_x, pad_y))) - the dataloader's `shapes[si]` (val.py:213,233).
    iouv: the IoU thresholds (val.py:165 torch.linspace(0.5, 0.95, 10)).
    Returns (correct [B, max_det, niou] bool, pred_polyn [B, max_det, 8], pred_hbbn [B, max_det, 4]); rows >= counts[b] are
    unspecified for the geometry and False for `correct`.  Everything stays on the device; no synchronisation."""
    _lib.require_cuda(dets, "dets")
    B, max_det, _ = dets.shape
    dev = dets.device
    d = dets.detach().float().contiguous()
    cnt = counts.detach().to(torch.int64).contiguous()
    tg = targets.detach().float()[:, :7].contiguous() if targets.numel() else torch.zeros((0, 7), device=dev)
    sc = torch.tensor([[float(s[1][0][0]), float(s[1][1][0]), float(s[1][1][1]), float(s[0][0]), float(s[0][1])] for s in shapes],
                      dtype=torch.float32).to(dev)
    iv = iouv.detach().float().contiguous().to(dev)
    correct = torch.empty((B, max_det, iv.numel()), dtype=torch.uint8, device=dev)
    polyn = torch.empty((B, max_det, 8), dtype=torch.float32, device=dev) if want_geometry else None
    hbbn = torch.empty((B, max_det, 4), dtype=torch.float32, device=dev) if want_geometry else None
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().y5obb_val_match_f32(d.data_ptr(), cnt.data_ptr(), B, max_det, _lib.ptr(tg) if tg.numel() else None,
                                            tg.shape[0], sc.data_ptr(), iv.data_ptr(), iv.numel(), correct.data_ptr(),
                                            _lib.ptr(polyn), _lib.ptr(hbbn), flag.data_ptr(), _lib.stream_ptr(dev))
    _lib.check(rc, "y5obb_val_match_f32")
    return correct.bool(), polyn, hbbn
