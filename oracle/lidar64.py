"""Float64 restatement of the StreetSurf LiDAR loss and its adjoint.  TEST INFRASTRUCTURE.

Restates, in numpy, what csrc/lidar_loss.cu computes: the validity mask with the `discard_toofar` assignment and the outlier discard
against the median error (app/loss/lidar.py LidarLoss.forward), the depth term l1 / l2_relative with the 'mean' reduction (DepthLoss;
nr3d_lib/models/loss/recon.py, loss/utils.py) and the `neus_unisim` line-of-sight term (LineOfSightLoss.fn_for_neus_unisim), with the
gradients to the rendered depth and to the volume-render weights vw (the mask held constant).

Every boolean decision -- mask_pred > thresh, gt > 0, gt <= discard_toofar, err > median * factor, |t - gt| > eps -- is taken on the
operands rounded as the kernel (and torch on fp32 tensors) rounds them when `decide` is np.float32, or in float64 with np.float64; the
values are float64 along those decisions.  The median is sorted(err)[R // 2] with NaN last, as torch.sort.
"""
import numpy as np

FN_TYPES = ("l1", "l2_relative")


def _mask_err(pred, mask_pred, gt, thresh, discard_toofar, decide):
    p, mp, g = (np.asarray(a, dtype=decide) for a in (pred, mask_pred, gt))
    mask = (mp > decide(thresh)) & (g > 0)
    if discard_toofar is not None and discard_toofar > 0:
        mask = g <= decide(discard_toofar)                 # the reference assigns: the first mask is dropped
    err = np.abs(p - g) * mask                             # rounded as the decisions' dtype: the median is taken over these
    return mask, err


def kth_smallest(v, k):
    """sorted(v)[k] with NaN last (torch.sort)"""
    return np.sort(np.asarray(v), kind="stable")[k]


def lidar_mask(pred, mask_pred, gt, *, thresh=1.0e-7, discard_toofar=None, median_factor=100.0, decide=np.float32):
    """-> (mask bool [R], err [R], median or None)"""
    mask, err = _mask_err(pred, mask_pred, gt, thresh, discard_toofar, decide)
    med = None
    if median_factor > 0:
        med = kth_smallest(err, err.shape[0] // 2)
        mask = mask & ~(err > decide(med) * decide(median_factor))
    return mask, err, med


def depth_term(pred, gt, mask, fn_type, w):
    """-> (w sum f mask / R, d/d pred)"""
    x, y, m = np.asarray(pred, np.float64), np.asarray(gt, np.float64), np.asarray(mask, np.float64)
    R = x.shape[0]
    d = x - y
    if fn_type == "l1":
        f, df = np.abs(d), np.sign(d)
    elif fn_type == "l2_relative":
        den = x * x + 1e-2
        f = d * d / den
        df = 2 * d / den - (d * d / (den * den)) * 2 * x
    else:
        raise ValueError(fn_type)
    return w * float(np.sum(f * m)) / R, w * df * m / R


def los_term(t, vw, pack_infos, rays_inds_hit, gt, mask, eps, w, decide=np.float32):
    """-> (w mean over kept rays of mask sum [|t - gt| > eps] vw^2 (0 with no kept ray), d/d vw [K], per-ray sums [n_hit])"""
    t, vw, gt = np.asarray(t), np.asarray(vw, np.float64), np.asarray(gt)
    pi, rih = np.asarray(pack_infos, np.int64), np.asarray(rays_inds_hit, np.int64)
    n_hit = pi.shape[0]
    g_vw = np.zeros(vw.shape[0], np.float64)
    rows = np.zeros(n_hit, np.float64)
    for p in range(n_hit):
        b, n, r = int(pi[p, 0]), int(pi[p, 1]), int(rih[p])
        sel = np.abs(t[b:b + n].astype(decide) - decide(gt[r])) > decide(eps)
        m = float(mask[r])
        rows[p] = m * float(np.sum(sel * vw[b:b + n] ** 2))
        g_vw[b:b + n] = w / n_hit * m * sel * 2 * vw[b:b + n]
    return (w * float(rows.sum()) / n_hit if n_hit else 0.0), g_vw, rows


def lidar_loss(pred, mask_pred, gt, t=None, vw=None, pack_infos=None, rays_inds_hit=None, *, fn_type="l1", w_depth=1.0, w_los=None, epsilon=1.0,
               thresh=1.0e-7, discard_toofar=None, median_factor=100.0, decide=np.float32):
    """LidarLoss.forward and its adjoint -> dict(depth, los (None without w_los), mask, median, g_depth, g_vw)"""
    mask, _, med = lidar_mask(pred, mask_pred, gt, thresh=thresh, discard_toofar=discard_toofar, median_factor=median_factor, decide=decide)
    out = dict(mask=mask, median=med, depth=None, g_depth=None, los=None, g_vw=None)
    if fn_type is not None:
        out["depth"], out["g_depth"] = depth_term(pred, gt, mask, fn_type, w_depth)
    if w_los is not None:
        out["los"], out["g_vw"], _ = los_term(t, vw, pack_infos, rays_inds_hit, gt, mask, epsilon, w_los, decide=decide)
    return out
