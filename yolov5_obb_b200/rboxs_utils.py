"""Host-side mirror of utils/rboxs_utils.py (tensor branches) and general.scale_polys, backed
by csrc/rbox_utils.cu: rbox2poly (:106-126), poly2hbb (:147-165), gaussian_label (:9-26, on the device so
that only [nt,7] targets need to cross PCIe — SURVEY §8f rank 2), scale_polys (utils/general.py:636-650)."""
import torch

from . import _lib

pi = 3.141592  # utils/rboxs_utils.py:5


def _run(fn, what, dev, *args):
    with torch.cuda.device(dev):
        rc = fn(*args, _lib.stream_ptr(dev))
    _lib.check(rc, what)


def rbox2poly(obboxes: torch.Tensor) -> torch.Tensor:
    """(num_gts, [cx cy l s θ]) θ∈[-pi/2, pi/2) -> (num_gts, [x1 y1 x2 y2 x3 y3 x4 y4])."""
    _lib.require_cuda(obboxes, "obboxes")
    lead = obboxes.shape[:-1]
    r = obboxes.reshape(-1, 5).float().contiguous()
    out = torch.empty((r.shape[0], 8), dtype=torch.float32, device=r.device)
    _run(_lib.lib().y5obb_rbox2poly_f32, "y5obb_rbox2poly_f32", r.device, r.data_ptr(), out.data_ptr(), r.shape[0])
    return out.reshape(*lead, 8)


def poly2hbb(polys: torch.Tensor) -> torch.Tensor:
    """(num_gts, poly) -> (num_gts, [xc yc w h])."""
    _lib.require_cuda(polys, "polys")
    assert polys.shape[-1] == 8
    p = polys.reshape(-1, 8).float().contiguous()
    out = torch.empty((p.shape[0], 4), dtype=torch.float32, device=p.device)
    _run(_lib.lib().y5obb_poly2hbb_f32, "y5obb_poly2hbb_f32", p.device, p.data_ptr(), out.data_ptr(), p.shape[0])
    return out


def scale_polys(img1_shape, polys: torch.Tensor, img0_shape, ratio_pad=None) -> torch.Tensor:
    """Rescale polys (xyxyxyxy) from img1_shape to img0_shape, in place (utils/general.py:636-650)."""
    _lib.require_cuda(polys, "polys")
    if ratio_pad is None:
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    else:
        gain = ratio_pad[0][0]
        pad = ratio_pad[1]
    if polys.dtype != torch.float32 or not polys.is_contiguous() or polys.shape[-1] != 8:
        raise RuntimeError("scale_polys works in place on a contiguous fp32 [n,8] tensor")
    _run(_lib.lib().y5obb_scale_polys_f32, "y5obb_scale_polys_f32", polys.device, polys.data_ptr(),
         polys.numel() // 8, float(pad[0]), float(pad[1]), float(gain))
    return polys


def gaussian_label(angle_deg: torch.Tensor, num_class: int = 180, u=0, sig: float = 4.0) -> torch.Tensor:
    """Batched gaussian_label_cpu: angles (degrees, θ·180/pi + 90) -> [n, num_class] fp32 CSL rows."""
    _lib.require_cuda(angle_deg, "angle_deg")
    assert u == 0
    a = angle_deg.reshape(-1).double().contiguous()
    out = torch.empty((a.shape[0], num_class), dtype=torch.float32, device=a.device)
    _run(_lib.lib().y5obb_gaussian_label, "y5obb_gaussian_label", a.device, a.data_ptr(), out.data_ptr(), a.shape[0],
         int(num_class), float(sig))
    return out


def poly2rbox(polys: torch.Tensor, num_cls_thata: int = 180, radius: float = 6.0, use_pi: bool = False,
              use_gaussian: bool = False):
    """utils/rboxs_utils.py:39-81 on the device: (num_gts, [x1 y1 x2 y2 x3 y3 x4 y4]) -> (num_gts, [cx cy l s theta]) fp64,
    theta in [-pi/2, pi/2) (use_pi) or degrees in [0, 180); with use_gaussian also the (num_gts, num_cls_thata) CSL rows
    (gaussian_label_cpu(label=angle_deg, u=0, sig=radius)).  The reference's arithmetic is cv2.minAreaRect; see
    csrc/rbox_utils.cu k_poly2rbox for the restated algorithm and tests/test_rbox_gpu.py for the parity statement."""
    _lib.require_cuda(polys, "polys")
    assert polys.shape[-1] == 8
    p = polys.reshape(-1, 8).float().contiguous()   # np.float32(poly), rboxs_utils.py:60
    out = torch.empty((p.shape[0], 5), dtype=torch.float64, device=p.device)
    _run(_lib.lib().y5obb_poly2rbox, "y5obb_poly2rbox", p.device, p.data_ptr(), out.data_ptr(), p.shape[0], int(bool(use_pi)))
    if not use_gaussian:
        return out
    angle = out[:, 4] if not use_pi else out[:, 4] * 180 / pi + 90
    return out, gaussian_label(angle, num_cls_thata, 0, radius)
