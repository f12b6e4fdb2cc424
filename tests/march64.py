"""What the occupancy-grid marcher's samples mean, checked in float64 without the C oracle's reading of the fp32 rounding sequence.

Sample counts depend on that sequence, so float64 cannot reproduce them bit for bit; it can check the meaning (nr3d_lib's
ray_marching.cu / batched_marching.cu, helpers_march.h):
  * layout: packed_info is the exclusive scan of the counts, ridx (and bidx) name the sample's ray (and batch), count <= max_steps;
  * each sample's midpoint t_mid = (t_start + t_end) / 2 lies before far, in the roi, in an occupied voxel, and that voxel is gidx
    (flat over [B, X, Y, Z] for the batched march); t_mid increases within a ray;
  * samples are contiguous through occupied space: when a sample does not start where the previous one ended, the step that would
    have followed the previous one ends in an empty voxel or outside the roi;
  * no occupied voxel is skipped: a float64 3-D DDA walk lists the voxels the ray crosses, and every occupied voxel with a chord
    longer than 2 dt + dt_min (dt: the step length calc_dt gives at the voxel's exit, at most dt_max) that lies before the ray's last
    sample (before far if the ray did not reach max_steps) holds a sample.
Points within `tol` of a voxel or roi face are exempt from the voxel checks.  t values are fp32 as the marcher's, so the midpoint and the
step that follows a sample are formed in fp32 (the source's own expressions), and only the point along the ray is taken in float64."""
import numpy as np

f32 = np.float32


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def _calc_dt(t, dt_gamma, dt_min, dt_max):
    return np.minimum(np.maximum(t * f32(dt_gamma), f32(dt_min)), f32(dt_max)).astype(f32)


def _locate(p, lo, hi, res, tol):
    """-> (flat voxel index, inside the roi, within tol of a voxel or roi face) of float64 points p [N, 3] in rois lo / hi [N, 3]"""
    res = np.asarray(res)
    vox = (hi - lo) / res
    u = (p - lo) / vox
    near = (np.abs(u - np.round(u)) * vox < tol).any(-1)
    inside = ((p >= lo) & (p <= hi)).all(-1)
    c = np.clip(np.floor(u), 0, res - 1).astype(np.int64)
    return (c[:, 0] * res[1] + c[:, 1]) * res[2] + c[:, 2], inside, near


def _walk(o, d, t_lo, t_hi, lo, hi, res):
    """float64 DDA: -> (ray, flat voxel, t_in, t_out) of every voxel each ray crosses between t_lo and t_hi inside the roi lo / hi"""
    res = np.asarray(res)
    vox = (hi - lo) / res
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = (lo - o) / d, (hi - o) / d
        ta = np.where(d != 0, ta, -np.inf); tb = np.where(d != 0, tb, np.inf)
    t_in = np.maximum(t_lo, np.minimum(ta, tb).max(-1))
    t_in[((d == 0) & ((o < lo) | (o > hi))).any(-1)] = np.inf          # parallel to a slab it lies outside of
    t_out = np.minimum(t_hi, np.maximum(ta, tb).min(-1))
    live = np.nonzero(t_in < t_out)[0]
    t, t_end = t_in[live], t_out[live]
    # the entry point can sit on a face: take the voxel the ray enters (a hair inside along d)
    c = np.clip(np.floor((o[live] + (t + 1e-9 * (t_end - t))[:, None] * d[live] - lo[live]) / vox[live]), 0, res - 1).astype(np.int64)
    step = np.sign(d[live]).astype(np.int64)
    out = []
    while live.size:
        oo, dd, ll, vv = o[live], d[live], lo[live], vox[live]
        with np.errstate(divide="ignore", invalid="ignore"):
            tn = np.where(dd != 0, (ll + (c + (dd > 0)) * vv - oo) / dd, np.inf)
        ax = np.argmin(tn, -1)
        te = np.minimum(tn[np.arange(live.size), ax], t_end)
        out.append((live, (c[:, 0] * res[1] + c[:, 1]) * res[2] + c[:, 2], t, te))
        c[np.arange(live.size), ax] += step[np.arange(live.size), ax]
        keep = (te < t_end) & ((c >= 0) & (c < res)).all(-1)
        live, t, t_end, c, step = live[keep], te[keep], t_end[keep], c[keep], step[keep]
    if not out:
        e = np.zeros(0, np.int64)
        return e, e, np.zeros(0), np.zeros(0)
    return tuple(np.concatenate(x) for x in zip(*out))


def check(rays_o, rays_d, near, far, roi, grid, step_size, max_step_size, dt_gamma, max_steps, info, t_starts, t_ends, ridx, gidx,
          batch_inds=None, bidx=None, tol=1e-6):
    """asserts the properties above of one march's outputs (batched when batch_inds is given: grid [B, X, Y, Z], roi [B, 6])"""
    o, d = _np(rays_o).astype(np.float64), _np(rays_d).astype(np.float64)
    near, far = _np(near).astype(f32), _np(far).astype(f32)
    info, ridx, gidx = _np(info).astype(np.int64), _np(ridx).astype(np.int64), _np(gidx).astype(np.int64)
    t0, t1 = _np(t_starts).reshape(-1).astype(f32), _np(t_ends).reshape(-1).astype(f32)
    g = _np(grid).astype(bool)
    batched = batch_inds is not None
    roi = _np(roi).astype(np.float64).reshape(-1, 6)
    res = g.shape[-3:]
    cells = int(np.prod(res))
    R, M = o.shape[0], t0.shape[0]
    cnt = info[:, 1]
    # ---- layout
    assert (cnt >= 0).all() and (cnt <= max_steps).all(), "count outside [0, max_steps]"
    assert int(cnt.sum()) == M and np.array_equal(info[:, 0], np.cumsum(cnt) - cnt), "packed_info is not the scan of the counts"
    ray = np.repeat(np.arange(R), cnt)
    assert np.array_equal(ridx, ray), "ridx does not name the sample's ray"
    b = _np(batch_inds).astype(np.int64)[ray] if batched else np.zeros(M, np.int64)
    if batched:
        assert np.array_equal(_np(bidx).astype(np.int64), b), "bidx does not name the sample's batch"
    local = gidx - b * cells
    assert ((local >= 0) & (local < cells)).all(), "gidx is not flat over [B, X, Y, Z] at the sample's batch"
    assert g.reshape(-1)[b * cells + local].all(), "a sample's gidx names an empty voxel"
    # ---- order and range
    tm = ((t0 + t1) * f32(0.5)).astype(f32)
    assert (t1 > t0).all() and (tm < far[ray]).all(), "a sample ends before it starts, or its midpoint is not before far"
    same = ray[1:] == ray[:-1]
    assert (tm[1:][same] > tm[:-1][same]).all(), "t_mid does not increase within a ray"
    # ---- each sample's midpoint lies in the voxel gidx names
    lo, hi = roi[b, :3], roi[b, 3:]
    p = o[ray] + tm.astype(np.float64)[:, None] * d[ray]
    v, inside, exempt = _locate(p, lo, hi, res, tol)
    assert inside[~exempt].all(), "a sample's midpoint lies outside the roi"
    assert np.array_equal(v[~exempt], local[~exempt]), "a sample's midpoint is not in the voxel gidx names"
    # ---- contiguity: after a gap, the step that would have followed the previous sample ends in an empty voxel or outside the roi
    k = np.nonzero(same & (t0[1:] != t1[:-1]))[0]
    tn0 = t1[k]
    tn1 = (tn0 + _calc_dt(tn0, dt_gamma, step_size, max_step_size)).astype(f32)
    tmn = ((tn0 + tn1) * f32(0.5)).astype(f32)
    bk = b[k]
    pn = o[ray[k]] + tmn.astype(np.float64)[:, None] * d[ray[k]]
    vn, inn, exn = _locate(pn, roi[bk, :3], roi[bk, 3:], res, tol)
    occ = inn & g.reshape(-1)[bk * cells + vn]
    assert not (occ & ~exn).any(), "samples skip over a step in an occupied voxel"
    # ---- no occupied voxel is skipped
    last = info[:, 0] + cnt - 1
    horizon = np.where(cnt == max_steps, tm[np.maximum(last, 0)] if M else 0, far).astype(np.float64)
    rb = _np(batch_inds).astype(np.int64) if batched else np.zeros(R, np.int64)
    wr = np.nonzero(rb >= 0)[0]                                  # rays with a negative batch index march nothing
    r_, vx, ti, to = _walk(o[wr], d[wr], near[wr].astype(np.float64), horizon[wr], roi[rb[wr], :3], roi[rb[wr], 3:], res)
    r_ = wr[r_]
    pm = o[r_] + ((ti + to) * 0.5)[:, None] * d[r_]             # a chord that runs along a voxel face (within tol) is exempt
    _, _, along_face = _locate(pm, roi[rb[r_], :3], roi[rb[r_], 3:], res, tol)
    long_chord = to - ti > 2 * np.clip(dt_gamma * to, step_size, max_step_size) + step_size
    need = g.reshape(-1)[rb[r_] * cells + vx] & long_chord & (to < horizon[r_]) & ~along_face
    have = np.unique(ray * (len(roi) * cells) + gidx)
    miss = ~np.isin(r_[need] * (len(roi) * cells) + rb[r_[need]] * cells + vx[need], have)
    assert not miss.any(), f"{int(miss.sum())} occupied voxels with a long chord hold no sample"
    return dict(samples=M, exempt=int(exempt.sum()), gaps=int(k.size), walked=int(need.sum()))
