"""Float64 restatement of the numerics contract of the per-ray NeuS stage kernels.  TEST INFRASTRUCTURE.

Covers k_upsample_cdf, k_invert_cdf_shared_u, k_neus_alpha_fwd / k_neus_alpha_bwd and k_composite_fwd / k_composite_bwd
(neuralsim_b200/csrc/neus_fused.cu) and the device functions of csrc/neus_device.cuh they share with k_upsample_persistent.
Every index-valued result is decided by an fp32 replay (numpy float32, one rounded operation at a time, in the order of the
reference's serial loop); every value is then float64 along those decisions.  What separates a kernel from this reference is only
CUDA's expf (not correctly rounded), fp32 rounding of plain sums and products, and their summation order.

fp32 decision points (names as in the kernels):
  x        = fl32(sdf * inv_s): the sigmoid argument of neus_alpha_at / k_neus_alpha_bwd (the values below use sigmoid(x) in float64)
  replay   the transmittance recurrence of packed_alpha_to_vw (pack_ops_cuda.cu:1736-1848, replay_chunk): before every sample
           `T < eps` stops the pack; the forward skips alpha <= thre, the backward skips alpha < thre (so at alpha == thre the
           backward visits the sample and multiplies T by 1 - alpha where the forward did not); w = fl32(alpha T),
           T = fl32(T fl32(1 - alpha)).  Replayed from the kernel's own alphas, so selector, num_steps and vw are bit-comparable.
  clamp    raw >= 0 of alpha = max(raw, 0): the alpha backward passes d_alpha only where the interval's raw alpha is >= 0
           (ATen's clamp_min rule); decided here from x_k >= x_{k+1} (sigmoid is monotone)
  cdf      norm = max(last exclusive cdf, 1e-5)
  invert   the lower bound over the pack's fp32 cdf (`cdf < u`), clamped to n - 1; pmf = fl32(cdf[pos] - cdf[pos-1]) < 1e-5 picks
           bins[pos-1]; pos == 0 picks bins[0].  An empty pack has no bin: the kernel writes NaN and reads nothing.
  estimate the slope clamp min(max(min(prev, dot), -10), 0) of neus_packed_sdf_to_upsample_alpha, evaluated in float64

Values (float64 along the decisions): alpha and the up-sampling estimate alpha (packed_diff's trailing zero: the last sample of
a pack has alpha 0; its first has prev slope 0), the exclusive cdf, mask / depth (normalised or not) / rgb / nablas sums,
the inverse-cdf sample, and the two backward passes written by hand:
  composite   g_w = g_mask + g_depth (t - D) / (M + 1e-10) [or g_depth t] + g_vw + g_rgb . rgb + g_nab . nablas;
              for every sample the backward visits: d_alpha_k = (g_w,k T_k - sum_{j>=k} g_w,j w_j) / max(1 - alpha_k, 1e-10),
              zero for skipped samples and after the stop;  d_rgb = w g_rgb, d_nablas = w g_nab
  alpha       c = sigmoid(x);  d c_k = [k < n-1][raw_k >= 0] g_k (c_{k+1} + 1e-5) / (c_k + 1e-5)^2
                                    - [k > 0][raw_{k-1} >= 0] g_{k-1} / (c_{k-1} + 1e-5)
              d_sdf = d c c (1 - c) inv_s;  d_inv_s = sum d c c (1 - c) sdf
tests/test_neus64_oracle.py checks the hand-written backward passes against torch float64 autograd, the replay against
oracle/pack_ops.py bit for bit, and the float64 values against oracle/render.py.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24            # unit roundoff of fp32 (half an ulp of 1)


def _sig(x):
    """sigmoid in float64, accurate in relative terms on both tails (so is c (1 - c) = _sig(x) _sig(-x))"""
    x = np.asarray(x, dtype=np.float64)
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def rows(pack_infos):
    """pack_infos [P,2] -> (idx [P,N] int64 of each pack's samples (0 where padded), valid [P,N]); N = the longest pack (>= 1)"""
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    N = max(int(pi[:, 1].max()) if pi.shape[0] else 0, 1)
    j = np.arange(N)
    valid = j[None, :] < pi[:, 1:2]
    return np.where(valid, pi[:, 0:1] + j[None, :], 0), valid


def pack_of(pack_infos, S):
    """sample -> pack index (-1 for samples no pack covers)"""
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    out = np.full(S, -1, dtype=np.int64)
    idx, valid = rows(pi)
    out[idx[valid]] = np.nonzero(valid)[0]
    return out


# ============================================================================================================ fp32 decisions
def replay(alpha, pack_infos, eps, thre, backward=False):
    """The serial fp32 transmittance recurrence of every pack, vectorised over packs.
    alpha [S] (fp32 values).  -> dict of
      vis [S] bool: the sample changes T (forward: alpha > thre; backward: alpha >= thre) and comes before the stop
      w [S] f32: alpha T at visited samples (forward only; the selector is vis), 0 elsewhere
      T [S] f32: T when the loop reaches the sample (samples after the stop: the T at the stop)
      steps [P]: visited samples;  stop [P]: the first sample before which T < eps (n if none)
      cross [P]: the visited sample after which T fell below eps (-1 if none);  T_end [P]"""
    a = np.asarray(alpha, dtype=F32)
    S = a.shape[0]
    idx, valid = rows(pack_infos)
    P, N = idx.shape
    A = np.where(valid, a[idx], F32(0))
    eps, thre, one = F32(eps), F32(thre), F32(1)
    T = np.ones(P, dtype=F32)
    stopped = np.zeros(P, dtype=bool)
    stop = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)[:, 1].copy()
    cross = np.full(P, -1, dtype=np.int64)
    VIS, W, TB = np.zeros((P, N), bool), np.zeros((P, N), F32), np.zeros((P, N), F32)
    for j in range(N):
        live = valid[:, j] & ~stopped
        now = live & (T < eps)
        stop[now] = j
        stopped |= now
        live &= ~now
        TB[:, j] = T
        aj = A[:, j]
        v = live & ((aj >= thre) if backward else (aj > thre))
        VIS[:, j] = v
        W[:, j] = np.where(v, aj * T, F32(0))
        Tn = np.where(v, T * (one - aj), T)
        cross[v & (T >= eps) & (Tn < eps)] = j
        T = Tn
    vis, w, Tb = np.zeros(S, bool), np.zeros(S, F32), np.zeros(S, F32)
    vis[idx[valid]], w[idx[valid]], Tb[idx[valid]] = VIS[valid], W[valid], TB[valid]
    return dict(vis=vis, w=w, T=Tb, steps=VIS.sum(1), stop=stop, cross=cross, T_end=T)


def compression(steps):
    """pack infos of the compressed packs (packed_volume_render_compression): (nidx, [first, count])"""
    steps = np.asarray(steps, dtype=np.int64)
    nidx = np.nonzero(steps > 0)[0]
    kept = steps[nidx]
    return nidx, np.stack([np.cumsum(kept) - kept, kept], 1)


def sigmoid_arg(sdf, inv_s):
    """x = fl32(sdf * inv_s): the kernels' first rounding"""
    return (np.asarray(sdf, dtype=F32) * F32(inv_s)).astype(F32)


# ============================================================================================================ float64 values
def neus_alpha(sdf, pack_infos, inv_s):
    """neus_alpha_at in float64 from x = fl32(sdf inv_s).  -> (alpha [S], scale [S]): scale = (c_k + c_{k+1}) / (c_k + 1e-5), the sum
    of the magnitudes the fp32 kernel subtracts (its error is a few fp32 ulps of it)"""
    x = sigmoid_arg(sdf, inv_s)
    c = _sig(x)
    S = c.shape[0]
    last = _last_mask(pack_infos, S)
    c1 = np.where(last, 0.0, np.roll(c, -1))
    raw = np.where(last, 0.0, (c - c1) / (c + 1e-5))
    scale = np.where(last, 0.0, (c + c1) / (c + 1e-5))
    return np.maximum(raw, 0.0), scale


def _last_mask(pack_infos, S):
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    m = np.zeros(S, dtype=bool)
    pi = pi[pi[:, 1] > 0]
    m[pi[:, 0] + pi[:, 1] - 1] = True
    return m


def _first_mask(pack_infos, S):
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    m = np.zeros(S, dtype=bool)
    pi = pi[pi[:, 1] > 0]
    m[pi[:, 0]] = True
    return m


def upsample_alpha(sdf, depth, pack_infos, inv_s):
    """neus_packed_sdf_to_upsample_alpha (neus_utils.py:164-188) in float64: interval k = [k, k+1], the last one has sdf_diff = delta = 0;
    prev slope of the first sample is 0; slope = min(max(min(prev, dot), -10), 0)"""
    s, d = np.asarray(sdf, np.float64), np.asarray(depth, np.float64)
    S = s.shape[0]
    last, first = _last_mask(pack_infos, S), _first_mask(pack_infos, S)
    ds = np.where(last, 0.0, np.roll(s, -1) - s)
    dt = np.where(last, 0.0, np.roll(d, -1) - d)
    dot = ds / (dt + 1e-5)
    prev = np.where(first, 0.0, np.roll(dot, 1))
    slope = np.minimum(np.maximum(np.minimum(prev, dot), -10.0), 0.0)
    mid = s + 0.5 * ds
    c0 = _sig((mid - 0.5 * slope * dt) * float(inv_s))
    c1 = _sig((mid + 0.5 * slope * dt) * float(inv_s))
    return np.maximum((c0 - c1) / (c0 + 1e-5), 0.0)


def transmittance(alpha, vis, pack_infos):
    """float64 T before each sample and w = alpha T along fixed decisions (vis: the samples that multiply T)"""
    a = np.asarray(alpha, np.float64)
    idx, valid = rows(pack_infos)
    f = np.where(valid & vis[idx], 1.0 - a[idx], 1.0)
    Tr = np.cumprod(np.concatenate([np.ones((idx.shape[0], 1)), f[:, :-1]], 1), 1)
    T = np.zeros(a.shape[0])
    T[idx[valid]] = Tr[valid]
    return T, np.where(vis, a * T, 0.0)


def upsample_cdf(w, pack_infos):
    """normalised exclusive cdf of weights w [S] (float64): cdf_k = sum_{j<k} w_j / max(sum_{j<n-1} w_j, 1e-5).
    -> (cdf [S], scale [S]: the magnitude behind each fp32 value, (5 + chunks) (sum_{j<=k} |w_j| + |cdf_k| sum_j |w_j|) / norm + |cdf_k|)"""
    w = np.asarray(w, np.float64)
    idx, valid = rows(pack_infos)
    Wr = np.where(valid, w[idx], 0.0)
    excl = np.cumsum(Wr, 1) - Wr
    n = valid.sum(1)
    last = excl[np.arange(idx.shape[0]), np.maximum(n - 1, 0)]
    norm = np.maximum(last, 1e-5)[:, None]
    # the kernel's exclusive value is (warp scan + carry) - w_k: a sum over j <= k, rounded once per scan level and once per chunk's
    # carry; the norm is the same sum over the pack
    absi = np.cumsum(np.abs(Wr), 1)
    depth = 5 + -(-n // 32)[:, None]
    c = excl / norm
    cdf, scale = np.zeros(w.shape[0]), np.zeros(w.shape[0])
    cdf[idx[valid]] = c[valid]
    scale[idx[valid]] = (depth * (absi + np.abs(c) * absi[np.arange(idx.shape[0]), np.maximum(n - 1, 0)][:, None]) / norm + np.abs(c))[valid]
    return cdf, scale


def lower_bound(cc, u):
    """binary_search_unsafe (pack_ops_cuda.cu:1336-1363) with its probe sequence, for every u at once: the first i with !(cc[i] < u)
    (an fp32 cumsum may step down by an ulp, so the probe order decides where it does)"""
    first = np.zeros(u.shape[0], np.int64)
    count = np.full(u.shape[0], cc.shape[0], np.int64)
    while (count > 0).any():
        step = count >> 1
        it = first + step
        lt = (count > 0) & (cc[np.minimum(it, cc.shape[0] - 1)] < u)
        first = np.where(lt, it + 1, first)
        count = np.where(lt, count - step - 1, np.where(count > 0, step, count))
    return first


def invert_cdf(bins, cdf32, u, pack_infos, return_pos=False):
    """k_invert_cdf_shared_u: u [n_s] shared by all packs; cdf32 the fp32 cdf the kernel reads (decisions on it are exact).
    -> (samples [P, n_s] float64 (NaN for an empty pack), scale [P, n_s]: |b0| + |b1 - b0|), and with return_pos also pos [P, n_s]: the
    bin each sample took (the lower bound clamped to n - 1; 0 for an empty pack)"""
    b32, c32, u32 = np.asarray(bins, F32), np.asarray(cdf32, F32), np.asarray(u, F32)
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    P, ns = pi.shape[0], u32.shape[0]
    out, scale, pos = np.full((P, ns), np.nan), np.zeros((P, ns)), np.zeros((P, ns), np.int64)
    for p, (b, n) in enumerate(pi):
        if n == 0:
            continue
        cc, bb = c32[b:b + n], b32[b:b + n]
        q = np.minimum(lower_bound(cc, u32), n - 1)
        pos[p] = q
        c0 = np.where(q > 0, cc[q - 1], F32(0))
        pmf = (cc[q] - c0).astype(F32)
        b0 = np.where(q > 0, bb[q - 1], bb[0]).astype(np.float64)
        b1 = bb[q].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            interp = b0 + (u32.astype(np.float64) - c0) / pmf.astype(np.float64) * (b1 - b0)
            r = np.where(q == 0, bb[0], np.where(pmf < F32(1e-5), b0, interp))
        out[p] = r
        scale[p] = np.abs(b0) + np.abs(b1 - b0)
    return (out, scale, pos) if return_pos else (out, scale)


def composite_forward(w, t, pack_infos, rgb=None, nablas=None, normalize_depth=True):
    """per-pack sums of weights w [S] in float64 -> dict(mask, depth, rgb, nablas) and the matching `*_scale` (sum of |terms|, divided by
    M + 1e-10 for the normalised depth)"""
    w = np.asarray(w, np.float64)
    t = np.asarray(t, np.float64)
    P = np.asarray(pack_infos).reshape(-1, 2).shape[0]
    S = w.shape[0]
    pk = pack_of(pack_infos, S)
    on = pk >= 0

    def psum(v):
        out = np.zeros((P,) + v.shape[1:])
        np.add.at(out, pk[on], v[on])
        return out
    M, sd, sda = psum(w), psum(w * t), psum(np.abs(w * t))
    r = dict(mask=M, mask_scale=psum(np.abs(w)))
    if normalize_depth:
        r["depth"] = sd / (M + 1e-10)
        r["depth_scale"] = (sda + np.abs(r["depth"]) * r["mask_scale"]) / (M + 1e-10)
    else:
        r["depth"], r["depth_scale"] = sd, sda
    for k, v in (("rgb", rgb), ("nablas", nablas)):
        if v is not None:
            v = np.asarray(v, np.float64)
            r[k], r[k + "_scale"] = psum(w[:, None] * v), psum(np.abs(w[:, None] * v))
    return r


def composite_backward(alpha, t, pack_infos, w, T, vis, mask, depth, *, rgb=None, nablas=None, g_mask=None, g_depth=None, g_rgb=None,
                       g_nablas=None, g_vw=None, ray_index=None, normalize_depth=True):
    """The adjoint of k_composite_fwd as the reference's kernel states it (pack_ops_cuda.cu:1795-1848).  w: the forward's weights; T, vis:
    the BACKWARD's transmittance and visited samples (replay(..., backward=True) or float64 along them); mask / depth: per pack, the values
    the backward reads; g_*: per output slot (ray_index[p], or p).  -> dict(d_alpha, d_rgb, d_nablas and `*_scale`: the bound magnitudes
    (|g_w,k T_k| + log2(n) sum_{j>=k} |g_w,j w_j|) / max(1 - alpha_k, 1e-10) and |w g|)"""
    a, t = np.asarray(alpha, np.float64), np.asarray(t, np.float64)
    w, T = np.asarray(w, np.float64), np.asarray(T, np.float64)
    pi = np.asarray(pack_infos, dtype=np.int64).reshape(-1, 2)
    S, P = a.shape[0], pi.shape[0]
    o = np.arange(P) if ray_index is None else np.asarray(ray_index, np.int64)
    pk = pack_of(pi, S)
    on = pk >= 0
    ok = np.where(on, o[np.maximum(pk, 0)], 0)
    z = lambda: np.zeros(S)
    M, D = np.asarray(mask, np.float64)[np.maximum(pk, 0)], np.asarray(depth, np.float64)[np.maximum(pk, 0)]
    gw, gwa = z(), z()
    if g_mask is not None:
        v = np.asarray(g_mask, np.float64)[ok]
        gw += v
        gwa += np.abs(v)
    if g_depth is not None:
        v = np.asarray(g_depth, np.float64)[ok] * ((t - D) / (M + 1e-10) if normalize_depth else t)
        gw += v
        gwa += np.abs(np.asarray(g_depth, np.float64)[ok]) * ((np.abs(t) + np.abs(D)) / (M + 1e-10) if normalize_depth else np.abs(t))
    if g_vw is not None:
        gw += np.asarray(g_vw, np.float64)
        gwa += np.abs(np.asarray(g_vw, np.float64))
    out = {}
    for k, v, g in (("rgb", rgb, g_rgb), ("nablas", nablas, g_nablas)):
        if v is None:
            continue
        v = np.asarray(v, np.float64)
        gg = np.zeros((S, 3)) if g is None else np.asarray(g, np.float64)[ok]
        gw += (gg * v).sum(1)
        gwa += np.abs(gg * v).sum(1)
        out["d_" + k] = np.where(on[:, None], w[:, None] * gg, 0.0)
        out["d_" + k + "_scale"] = np.abs(out["d_" + k])
    gw, gwa = np.where(on, gw, 0.0), np.where(on, gwa, 0.0)
    idx, valid = rows(pi)
    gww = np.where(valid, (gw * w)[idx], 0.0)
    acc = np.cumsum(gww[:, ::-1], 1)[:, ::-1]                  # sum_{j>=k} g_w,j w_j
    # the fp32 accum is a pack sum (log2 n roundings deep) that then loses one visited sample's term at a time: its error at sample k is
    # bounded by log2(n) A_0 + sum_{visited i<k} A_i, A_i = sum_{j>=i} |g_w,j w_j|
    acca = np.cumsum(np.where(valid, np.abs(gwa * w)[idx], 0.0)[:, ::-1], 1)[:, ::-1]
    vr = np.where(valid, vis[idx], False)
    drift = np.cumsum(np.where(vr, acca, 0.0), 1) - np.where(vr, acca, 0.0)
    n = np.maximum(valid.sum(1, keepdims=True), 2)
    ea = np.log2(n) * acca[:, :1] + drift
    accum, accum_a = z(), z()
    accum[idx[valid]], accum_a[idx[valid]] = acc[valid], np.broadcast_to(ea, acca.shape)[valid]
    den = np.maximum(1.0 - a, 1e-10)
    out["d_alpha"] = np.where(vis, (gw * T - accum) / den, 0.0)
    out["d_alpha_scale"] = np.where(vis, (gwa * np.abs(T) + accum_a) / den, 0.0)
    out["g_w"] = gw
    return out


def alpha_backward(sdf, pack_infos, inv_s, d_alpha):
    """The adjoint of neus_alpha_at (k_neus_alpha_bwd).  -> dict(d_sdf [S], d_sdf_scale [S], d_inv_s, d_inv_s_abs, d_inv_s_ambiguous,
    ambiguous): d_sdf_scale is inv_s (|dL/dc| terms) (c (1 - c) + c^2 + 2^-126 / 2^-24), the magnitude fp32 loses a few ulps of; d_inv_s_abs the sum of
    |terms| of d_inv_s; d_inv_s_ambiguous the absolute share of d_inv_s that ambiguous clamp decisions may add"""
    s = np.asarray(sdf, np.float64)
    g = np.asarray(d_alpha, np.float64)
    S = s.shape[0]
    x = sigmoid_arg(sdf, inv_s).astype(np.float64)
    c = _sig(x)
    last, first = _last_mask(pack_infos, S), _first_mask(pack_infos, S)
    covered = pack_of(pack_infos, S) >= 0
    c1 = np.roll(c, -1)
    act = ~last & covered & (x >= np.roll(x, -1))                  # raw_k >= 0 of interval k = [k, k+1]
    g_own = np.where(act, g, 0.0)
    t_own = g_own * (c1 + 1e-5) / (c + 1e-5) ** 2
    act_p, g_p, c_p = np.roll(act, 1) & ~first & covered, np.roll(g, 1), np.roll(c, 1)
    t_prev = np.where(act_p, g_p / (c_p + 1e-5), 0.0)
    gc = t_own - t_prev
    ga = np.abs(t_own) + np.abs(t_prev)
    dc = c * _sig(-x)
    # a rising interval whose two fp32 sigmoids round to the same value has raw == 0 in the kernel (clamp open): such an interval may
    # add its whole term, so it enters the bound in full (in units of 2^-24)
    cf = c.astype(F32)
    amb = ~last & covered & (x < np.roll(x, -1)) & (np.abs(c - c1) <= 2 * np.spacing(np.maximum(cf, np.roll(cf, -1))))
    e_own = np.where(amb, np.abs(g) * (c1 + 1e-5) / (c + 1e-5) ** 2, 0.0)
    e_prev = np.where(np.roll(amb, 1) & ~first, np.abs(g_p) / (c_p + 1e-5), 0.0)
    e_amb = (e_own + e_prev) * dc
    iv = float(F32(inv_s))
    terms = gc * dc * s
    # fp32 c (1 - c) carries an error of a few 2^-24 (dc + c^2): relative where c is small, absolute (1 - c rounds) where c is near 1;
    # below sigmoid(-88.7) expf overflows and c is 0 (an absolute error under 2^-126)
    dce = dc + c * c + 2.0 ** -126 / U32
    return dict(d_sdf=gc * dc * iv, d_sdf_scale=(ga * dce + e_amb / U32) * iv, d_inv_s=float(terms.sum()),
                d_inv_s_abs=float(np.abs(terms).sum()), d_inv_s_ambiguous=float((e_amb * np.abs(s)).sum()), ambiguous=int(amb.sum()))
