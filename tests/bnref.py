"""fp64 references and per-element error bounds for the training BatchNorm / SiLU / routing kernels (csrc/bn_train.cu).

Runs on any torch device.  The bounds restate the kernels' fp32 arithmetic:

  * Sums (k_bn_stats / k_bn_bwd_reduce, then k_reduce_partials / k_reduce_finalize): every term reaches the result through at
    most `stat_chain()` fp32 additions, so |fl(sum) - sum| <= gamma(d) * sum|term| with gamma(d) = d u / (1 - d u), u = 2^-24.
    The geometry (blocks, chunk, lanes, the 16-lane tree, the 32-segment reduce) is restated from bn_train.cu;
    `emulate_stats` replays the kernels' exact fp32 order on the CPU so the depth and the bound can be checked there.
  * SiLU: the sigmoid is 0.5 tanh.approx(u / 2) + 0.5.  PTX documents tanh.approx's relative error as 2^-10.987; the bounds use
    2^-10 (as tests/test_conv_plans_exact_gpu.py does), i.e. an absolute sigmoid error of at most 2^-11.
  * bf16 results are one round-to-nearest of an fp32 value: half a bf16 ulp of the exact value plus the fp32 error before it.
"""
import numpy as np
import torch

U = 2.0 ** -24                  # fp32 unit roundoff
TANH_REL = 2.0 ** -10           # tanh.approx.f32 relative error used in the bounds (PTX: 2^-10.987)
SIG_ERR = 0.5 * TANH_REL + U    # absolute error of sigmoid_tanh (0.5 * |tanh| * rel + the fma's rounding)
STAT_THREADS = 256


# ---------------------------------------------------------------------------------------------------------------- geometry
def stat_layout(C: int):
    """(vecs, cols, lanes) of k_bn_stats / k_bn_bwd_reduce: `cols` threads cover a pixel's 8-channel vectors, `lanes`
    pixels are in flight per block; C / 8 > 256 takes several column groups (the cv0 loop)."""
    vecs = C // 8
    cols = min(vecs, STAT_THREADS)
    return vecs, cols, STAT_THREADS // cols


def stat_blocks(npix: int, C: int, sms: int) -> int:
    """stat_blocks(): >= 16 pixels per thread, at most 4 blocks per SM."""
    lanes = stat_layout(C)[2]
    want = -(-npix // (lanes * 16))
    return max(1, min(want, 4 * sms))


def colwise_grid(npix: int, C: int, sms: int):
    """colwise_grid() of k_bn_silu_apply / k_bn_bwd_apply: (x blocks, y column groups).  A block steps over 2 * lanes pixels
    (two per thread), at most 8 blocks per SM; a y block per group of `cols` vector columns."""
    vecs, cols, lanes = stat_layout(C)
    return max(1, min(-(-npix // (2 * lanes)), 8 * sms)), -(-vecs // cols)


def stat_geometry(npix: int, C: int, sms: int):
    """(blocks, chunk, lanes) of one statistics launch."""
    blocks = stat_blocks(npix, C, sms)
    return blocks, -(-npix // blocks), stat_layout(C)[2]


def stat_chain(npix: int, C: int, sms: int) -> int:
    """Longest chain of fp32 additions from a pixel's term to the channel's sum: a lane adds its pixels in order (at most
    ceil(chunk / lanes)), lanes l < 16 add lanes l + 16, l + 32, ..., lane 0 adds lanes 1..15, a reduce thread adds every
    32nd block partial, thread 0 adds the 31 other segment sums."""
    blocks, chunk, lanes = stat_geometry(npix, C, sms)
    per_lane = -(-chunk // lanes)
    tree16 = -(-(lanes - 16) // 16) if lanes > 16 else 0
    tree0 = min(16, lanes) - 1
    return per_lane + tree16 + tree0 + -(-blocks // 32) + 31


def gamma(d: int) -> float:
    return d * U / (1.0 - d * U)


def emulate_stats(x: np.ndarray, sms: int):
    """k_bn_stats + k_reduce_partials in their exact fp32 order on the CPU.  x: [npix, C] values exact in bf16.
    -> (sum, sumsq, depth): fp32 sums per channel and the longest addition chain any term went through."""
    x = np.asarray(x, dtype=np.float32)
    npix, C = x.shape
    blocks, chunk, lanes = stat_geometry(npix, C, sms)
    f32 = np.float32
    part_s = np.zeros((blocks, C), f32)
    part_q = np.zeros((blocks, C), f32)
    part_d = np.zeros(blocks, np.int64)
    for b in range(blocks):
        p0, p1 = b * chunk, min(npix, (b + 1) * chunk)
        s = np.zeros((lanes, C), f32)
        q = np.zeros((lanes, C), f32)
        d = np.zeros(lanes, np.int64)
        for lane in range(lanes):
            for p in range(p0 + lane, p1, lanes):
                s[lane] = s[lane] + x[p]
                q[lane] = f32(np.float64(q[lane]) + np.float64(x[p]) * x[p])   # fmaf(f, f, q): one rounding
                d[lane] += 1
        for lane in range(min(16, lanes)):
            for l2 in range(lane + 16, lanes, 16):
                s[lane] = s[lane] + s[l2]
                q[lane] = q[lane] + q[l2]
                d[lane] = max(d[lane], d[l2]) + 1
        for l2 in range(1, min(16, lanes)):
            s[0] = s[0] + s[l2]
            q[0] = q[0] + q[l2]
            d[0] = max(d[0], d[l2]) + 1
        part_s[b], part_q[b], part_d[b] = s[0], q[0], d[0]
    seg_s = np.zeros((32, C), f32)
    seg_q = np.zeros((32, C), f32)
    seg_d = np.zeros(32, np.int64)
    for seg in range(32):
        for b in range(seg, blocks, 32):
            seg_s[seg] = seg_s[seg] + part_s[b]
            seg_q[seg] = seg_q[seg] + part_q[b]
            seg_d[seg] = max(seg_d[seg], part_d[b]) + 1
    ts, tq, td = seg_s[0].copy(), seg_q[0].copy(), seg_d[0]
    for seg in range(1, 32):
        ts = ts + seg_s[seg]
        tq = tq + seg_q[seg]
        td = max(td, seg_d[seg]) + 1
    return ts, tq, int(td)


# ----------------------------------------------------------------------------------------------------------- rounding
def ulp32(x: torch.Tensor) -> torch.Tensor:
    """fp32 ulp of |x| (fp64 in, fp64 out; normal range)."""
    _, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 24).clamp(min=-149))


def half_ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Half a bf16 ulp of |x|: the largest error of one round-to-nearest into bf16 (8 significand bits)."""
    _, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 9).clamp(min=-134))


# ----------------------------------------------------------------------------------------------------------- forward
def finalize_ref(s: torch.Tensor, q: torch.Tensor, n: int, eps: float):
    """k_reduce_finalize's statistics in fp64 from the kernel's own fp32 sums: (mean64, var64, invstd64)."""
    m = s.double() / n
    var = (q.double() / n - m * m).clamp(min=0)
    return m, var, 1.0 / torch.sqrt(var + float(np.float32(eps)))


def silu_parts(u: torch.Tensor):
    """(sigmoid, silu, silu') in fp64."""
    sg = torch.sigmoid(u)
    return sg, u * sg, sg + u * sg * (1 - sg)


def apply_ref(z: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, act: bool, res=None):
    """y = [res +] act(z * scale + shift) in fp64 from the kernel's own fp32 scale / shift, and its per-element bound:
    u's fma rounding, the sigmoid approximation (|u| SIG_ERR), the product's and the residual add's fp32 roundings, then
    one bf16 rounding.  z, res: [..., C] (any float dtype); scale, shift: [C]."""
    u = z.double() * scale.double() + shift.double()
    du = u.abs() * U
    if act:
        _, y, _ = silu_parts(u)
        err = u.abs() * SIG_ERR + 1.1 * du + U * y.abs()
    else:
        y, err = u, du
    if res is not None:
        y = y + res.double()
        err = err + U * (y.abs() + err)
    return y, err + half_ulp_bf16(y.abs() + err)


# ---------------------------------------------------------------------------------------------------------- backward
def du_ref(z: torch.Tensor, dy: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, act: bool):
    """du = dy * act'(z * scale + shift) in fp64 and the bound on the kernel's fp32 du: u's rounding (silu'' <= 0.5), the
    sigmoid error through silu' = s + u s (1 - s) (derivative in s: 1 + u (1 - 2 s)), silu_grad's own roundings, the product."""
    d = dy.double()
    if not act:
        return d, torch.zeros_like(d)
    u = z.double() * scale.double() + shift.double()
    _, _, g = silu_parts(u)
    du = d * g
    eg = 0.5 * u.abs() * U + SIG_ERR * (1 + u.abs()) + 4 * U * (1 + u.abs())
    return du, d.abs() * eg + U * du.abs()


def dz_ref(z, du, du_err, scale, mean, invstd, sum_du, sum_dux, n: int):
    """dz = scale (du - sum_du / N - xhat sum_dux / N), xhat = (z - mean) invstd, in fp64 from the kernel's own per-channel
    fp32 values, and its bound: du's error times scale, the roundings of k1..k3 = scale, -scale b, scale (mean b - sum_du / N)
    (b = invstd sum_dux / N) and of the two fmas, then one bf16 rounding."""
    sc, m, iv = scale.double(), mean.double(), invstd.double()
    S, Q = sum_du.double() / n, sum_dux.double() / n
    b = iv * Q
    zd = z.double()
    y = sc * (du - S - (zd - m) * b)
    err = sc.abs() * du_err + 8 * U * (sc.abs() * ((b * zd).abs() + (b * m).abs() + S.abs() + du.abs()) + y.abs())
    return y, err + half_ulp_bf16(y.abs() + err)


# ---------------------------------------------------------------------------------------------------------- routing
def upsample2x_bwd_ref(g2: torch.Tensor, old=None) -> torch.Tensor:
    """k_upsample2x_bwd in fp32, its order: ((g[2h,2w] + g[2h,2w+1]) + g[2h+1,2w]) + g[2h+1,2w+1] [+ old], one RN to bf16.
    g2: [B, 2H, 2W, C] bf16; old: [B, H, W, C] bf16 or None."""
    g = g2.float()
    a = g[:, 0::2, 0::2] + g[:, 0::2, 1::2]
    a = a + g[:, 1::2, 0::2]
    a = a + g[:, 1::2, 1::2]
    if old is not None:
        a = a + old.float()
    return a.bfloat16()


def maxpool5_route(x: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """Backward of a 5x5 / stride 1 / pad 2 max pool: every g[b,h,w,c] to the window's first maximum in row-major order
    (ATen's rule), summed in fp64.  x, g: [B, H, W, C] -> [B, H, W, C] fp64."""
    B, H, W, C = x.shape
    xn = x.double().permute(0, 3, 1, 2).contiguous()
    _, idx = torch.nn.functional.max_pool2d(xn, 5, 1, 2, return_indices=True)
    out = torch.zeros(B, C, H * W, dtype=torch.float64, device=x.device)
    out.scatter_add_(2, idx.view(B, C, H * W), g.double().permute(0, 3, 1, 2).reshape(B, C, H * W))
    return out.view(B, C, H, W).permute(0, 2, 3, 1)


def detect_grad_pack_ref(g: torch.Tensor, bn: int) -> torch.Tensor:
    """[B, na, H, W, no] fp32 -> [B, H, W, na * bn] bf16, anchor a at channels [a bn, a bn + no), padding channels 0."""
    B, na, H, W, no = g.shape
    out = torch.zeros(B, H, W, na, bn, dtype=torch.bfloat16, device=g.device)
    out[..., :no] = g.permute(0, 2, 3, 1, 4).bfloat16()
    return out.view(B, H, W, na * bn)
