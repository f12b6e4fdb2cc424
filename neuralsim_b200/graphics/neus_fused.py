"""Fused per-ray NeuS stages (csrc/neus_fused.cu): each function is ONE kernel launch and is numerically the same
computation as the chain of `nr3d_lib` calls named in its docstring, which stays available in `graphics.neus` /
`graphics.pack_ops` (the unfused chain is what the parity tests compare these against).

  upsample_cdf            neus_packed_sdf_to_(upsample_)alpha -> packed_alpha_to_vw -> packed_cumsum(exclusive) -> normalise
  sample_cdf_uniform      packed_sample_cdf(perturb=False)           (reference: graphics/raysample.py:38-61)
  neus_alpha_compress     neus_packed_sdf_to_alpha (autograd) + packed_volume_render_compression's selector pass
  composite               packed_alpha_to_vw + packed_sum/packed_div + products of the volume integration
                          (reference: app/renderers/single_volume_renderer.py:73-102), with its adjoint
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib as L

__all__ = ["upsample_cdf", "sample_cdf_uniform", "neus_alpha_compress", "neus_alpha_compact", "composite", "scan_counts", "merge_sorted_vals",
           "assemble_boundary", "march_lean", "upsample_rays", "block_order", "ray_block_order", "ray_test_aabb", "gather_rays", "gather_rays_backward", "scan_launch", "march_listed",
           "pack_occ_bits", "alpha_forward", "compact_samples"]

# `count=` of the launch functions below: None, or (cnt, k0[, k1]) -- the sizes live in the device count block cnt and the size arguments
# (and the buffers) are capacities (_lib.call)

_U_CACHE = {}


def _f32c(t):
    return t.detach().contiguous().float()


def _quantiles(n, dev):
    """linspace(0, 1, n + 2)[1:-1]: the shared u of the non-perturbed inverse-cdf sampling"""
    key = (n, dev)
    u = _U_CACHE.get(key)
    if u is None:
        u = _U_CACHE[key] = torch.linspace(0., 1., n + 2, device=dev, dtype=torch.float32)[1:-1].contiguous()
    return u


@torch.no_grad()
def upsample_cdf(sdf, depth, pack_infos, inv_s: float, use_estimate_alpha=False, early_stop_eps=1e-4, alpha_thre=0.0, *, count=None):
    sdf, depth = _f32c(sdf), _f32c(depth)
    cdf = torch.empty_like(sdf)
    L.call(L.lib().nsb_neus_upsample_cdf, "neus_upsample_cdf", L.ptr(sdf, "f32"), L.ptr(depth, "f32"), L.ptr(pack_infos, "i64"),
           L.c_i64(pack_infos.shape[0]), L.c_f32(inv_s), ctypes.c_int(1 if use_estimate_alpha else 0), L.c_f32(early_stop_eps),
           L.c_f32(alpha_thre), L.ptr(cdf), L.stream_ptr(), count=count)
    return cdf


@torch.no_grad()
def sample_cdf_uniform(bins, cdfs, pack_infos, num_to_sample: int, *, count=None):
    u = _quantiles(num_to_sample, bins.device)
    P = pack_infos.shape[0]
    out = torch.empty(P, num_to_sample, device=bins.device, dtype=torch.float32)
    L.call(L.lib().nsb_packed_invert_cdf_shared_u, "packed_invert_cdf_shared_u", L.ptr(bins, "f32"), L.ptr(cdfs, "f32"), L.ptr(u, "f32"),
           L.ptr(pack_infos, "i64"), L.c_i64(P), L.c_i32(num_to_sample), L.ptr(out), L.stream_ptr(), count=count)
    return out


def alpha_forward(sdf, pack_infos, inv_s, early_stop_eps, alpha_thre, *, count=None):
    """nsb_neus_alpha_forward: sdf [S] f32, inv_s f32 [1] -> (alpha [S], sel [S] bool (kept by the compression), steps [P] int32 (kept per pack))"""
    P = pack_infos.shape[0]
    alpha = torch.empty_like(sdf)
    sel = torch.empty(sdf.shape[0], dtype=torch.bool, device=sdf.device)
    steps = torch.empty(P, dtype=torch.int32, device=sdf.device)
    L.call(L.lib().nsb_neus_alpha_forward, "neus_alpha_forward", L.ptr(sdf, "f32"), L.ptr(pack_infos, "i64"), L.c_i64(P), L.ptr(inv_s, "f32"),
           L.c_f32(early_stop_eps), L.c_f32(alpha_thre), L.ptr(alpha), L.ptr(sel), L.ptr(steps), L.stream_ptr(), count=count)
    return alpha, sel, steps


class _NeusAlpha(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sdf, inv_s, pack_infos, early_stop_eps, alpha_thre):
        sdf_c, inv_c = _f32c(sdf), _f32c(inv_s).reshape(1)
        alpha, sel, steps = alpha_forward(sdf_c, pack_infos, inv_c, early_stop_eps, alpha_thre)
        ctx.save_for_backward(sdf_c, inv_c, pack_infos)
        ctx.inv_shape = inv_s.shape
        ctx.mark_non_differentiable(sel, steps)
        return alpha, sel, steps

    @staticmethod
    def backward(ctx, g_alpha, _gs, _gn):
        sdf_c, inv_c, pack_infos = ctx.saved_tensors
        g = g_alpha.contiguous().float()
        d_sdf = torch.empty_like(sdf_c)
        d_inv = torch.zeros(1, device=sdf_c.device, dtype=torch.float32)
        L.check(L.lib().nsb_neus_alpha_backward(L.ptr(sdf_c, "f32"), L.ptr(pack_infos, "i64"), L.c_i64(pack_infos.shape[0]),
                                                L.ptr(inv_c, "f32"), L.ptr(g, "f32"), L.ptr(d_sdf), L.ptr(d_inv), L.stream_ptr()),
                "neus_alpha_backward")
        return (d_sdf if ctx.needs_input_grad[0] else None, d_inv.reshape(ctx.inv_shape) if ctx.needs_input_grad[1] else None,
                None, None, None)


def neus_alpha_compress(sdf, inv_s, pack_infos, early_stop_eps=1e-4, alpha_thre=0.0):
    """-> (alpha [S] (differentiable wrt sdf, inv_s), nidx_useful, pack_infos_useful, pidx_useful)."""
    if not isinstance(inv_s, torch.Tensor):
        inv_s = torch.tensor(float(inv_s), device=sdf.device)
    alpha, sel, steps = _NeusAlpha.apply(sdf, inv_s, pack_infos, early_stop_eps, alpha_thre)
    pidx = sel.nonzero()[..., 0]
    nidx = (steps > 0).nonzero()[..., 0]
    kept = steps[nidx].long()
    cs = kept.cumsum(0)
    return alpha, nidx, torch.stack([cs - kept, kept], 1), pidx


class _GatherUnique(torch.autograd.Function):
    """out = the kernel-made gather `src[pidx]` (pidx unique); backward scatters into zeros with one launch."""

    @staticmethod
    def forward(ctx, src, pidx, gathered):
        ctx.save_for_backward(pidx)
        ctx.n = src.shape[0]
        return gathered

    @staticmethod
    def backward(ctx, g):
        pidx, = ctx.saved_tensors
        g = g.contiguous().float()
        d = torch.zeros(ctx.n, dtype=torch.float32, device=g.device)
        L.check(L.lib().nsb_scatter_f32(L.ptr(g, "f32"), L.ptr(pidx, "i64"), L.c_i64(pidx.shape[0]), L.ptr(d), L.stream_ptr()), "scatter_f32")
        return d, None, None


_SCAN_WS = []
_HOST_SLOTS = {}


def _host_slot():
    """(pinned int64[4] tensor, its numpy view, ticket counter) -- the scan kernel writes the two totals (+ one extra) and a ticket there and
    the host polls the ticket: a data-dependent size reaches Python without cudaMemcpy / cudaStreamSynchronize."""
    dev = torch.cuda.current_device()
    st = _HOST_SLOTS.get(dev)
    if st is None:
        t = torch.zeros(4, dtype=torch.int64).pin_memory()
        st = _HOST_SLOTS[dev] = [t, t.numpy(), 0]
    return st


def _scan_ws_bytes():
    if not _SCAN_WS:
        L.lib().nsb_scan_workspace_bytes.restype = ctypes.c_int64
        _SCAN_WS.append(int(L.lib().nsb_scan_workspace_bytes()))
    return _SCAN_WS[0]


def scan_launch(counts, totals, *, first=None, info2=None, index=None, pack=None, src=None, nz_src=None, extra=None, ticket=0, ws=None):
    """nsb_scan_counts: the totals go to `totals` (a device pointer: a count block slot, or the pinned host slot with a ticket); ws: a
    zero-filled workspace of _scan_ws_bytes() (None: a fresh one)"""
    if ws is None:
        ws = torch.zeros(_scan_ws_bytes(), dtype=torch.uint8, device=counts.device)
    P = L.ptr
    L.check(L.lib().nsb_scan_counts(P(counts, "i32"), L.c_i64(counts.shape[0]), P(first, allow_none=True), P(info2, allow_none=True),
                                    P(index, allow_none=True), P(pack, allow_none=True), P(src, "i64", allow_none=True), P(nz_src, allow_none=True),
                                    totals, P(extra, "i64", allow_none=True), L.c_i64(ticket), P(ws), L.stream_ptr()), "scan_counts")


@torch.no_grad()
def scan_counts(counts, *, want_first=False, want_info2=False, want_index=False, want_pack=False, src=None, extra=None):
    """One launch + ONE host read: exclusive scan of int32 counts and compaction of the non-zero entries.
    -> dict(total, n_nonzero, first?, info2?, index?, pack?, src?) with the compacted outputs already sliced."""
    n, dev = counts.shape[0], counts.device
    first = torch.empty(n, dtype=torch.int32, device=dev) if want_first else None
    info2 = torch.empty(n, 2, dtype=torch.int32, device=dev) if want_info2 else None
    index = torch.empty(n, dtype=torch.int64, device=dev) if want_index else None
    pack = torch.empty(n, 2, dtype=torch.int64, device=dev) if want_pack else None
    nz_src = torch.empty(n, dtype=torch.int64, device=dev) if src is not None else None
    slot = _host_slot()
    slot[2] += 1
    ticket = slot[2]
    scan_launch(counts, ctypes.c_void_p(slot[0].data_ptr()), first=first, info2=info2, index=index, pack=pack, src=src, nz_src=nz_src, extra=extra,
                ticket=ticket)
    host = slot[1]                                    # the one host wait: output sizes are data dependent.  Polling pinned memory, no driver call
    spins = 0
    while host[3] != ticket:
        spins += 1
        if spins > 2_000_000 and spins % 1_000_000 == 0:     # ~ seconds: surface a dead kernel instead of hanging
            torch.cuda.current_stream().synchronize()
            if host[3] != ticket:
                raise RuntimeError("scan_counts: the kernel finished without publishing its totals")
    total, nnz = int(host[0]), int(host[1])
    out = dict(total=total, n_nonzero=nnz, first=first, info2=info2, extra=[int(host[2])])
    out["index"] = index[:nnz] if index is not None else None
    out["pack"] = pack[:nnz] if pack is not None else None
    out["src"] = nz_src[:nnz] if nz_src is not None else None
    return out


@torch.no_grad()
def ray_block_order(pix, via, n_rays, pairs, row_len, *, count=None):
    """order[P]: the packs on pixels pix[via[p]] (via None: pix[p]; ascending, unique) in 8 x 4 pixel blocks, for the ray-tiled SDF
    query (csrc/neus_glue.cu: k_ray_block_order).  n_rays: the rays the ray test saw; pairs, row_len: device pointers to its int64
    neighbour-pair count and row length."""
    n = pix.shape[0] if via is None else via.shape[0]
    order = torch.empty(n, dtype=torch.int64, device=pix.device)
    L.call(L.lib().nsb_ray_block_order, "ray_block_order", L.ptr(pix, "i64"), L.ptr(via, "i64", allow_none=True), L.c_i64(n), L.c_i64(n_rays),
           pairs, row_len, L.ptr(order), L.stream_ptr(), count=count)
    return order


def block_order(pix, via, rays_row):
    """ray_block_order with the ray test's rays_row = (rays it saw, its int64[2] (neighbour pairs, row length))"""
    n_rays, pr = rays_row
    return ray_block_order(pix, via, n_rays, L.ptr(pr, "i64"), L.ptr(pr[1:], "i64"))


def ray_test_aabb(rays_o, rays_d, center3, radius3, near, far, pairs, row_len):
    """nsb_ray_test_aabb -> (o_n, d_n, near, far, flag) of every ray; the neighbour-pair count and the row length go to the device
    pointers pairs / row_len"""
    R, dev = rays_o.shape[0], rays_o.device
    o_n, d_n = torch.empty(R, 3, device=dev), torch.empty(R, 3, device=dev)
    nr, fr = torch.empty(R, device=dev), torch.empty(R, device=dev)
    flag = torch.empty(R, dtype=torch.int32, device=dev)
    L.check(L.lib().nsb_ray_test_aabb(L.ptr(rays_o.contiguous(), "f32"), L.ptr(rays_d.contiguous(), "f32"), L.c_i64(R), center3, radius3,
                                      ctypes.c_int(0 if near is None else 1), L.c_f32(0. if near is None else near),
                                      ctypes.c_int(0 if far is None else 1), L.c_f32(0. if far is None else far), L.ptr(o_n), L.ptr(d_n),
                                      L.ptr(nr), L.ptr(fr), L.ptr(flag), pairs, row_len, L.stream_ptr()), "ray_test_aabb")
    return o_n, d_n, nr, fr, flag


def gather_rays(idx, n, tested, out, extra=None, extra_c=None, *, count=None):
    """nsb_gather_rays: rows idx[:n] of tested = (o_n, d_n, near, far) (and of extra) into out = (o_c, d_c, near_c, far_c) (and extra_c)"""
    (o_n, d_n, nr, fr), (o_c, d_c, n_c, f_c), P = tested, out, L.ptr
    L.call(L.lib().nsb_gather_rays, "gather_rays", P(idx, "i64"), L.c_i64(n), P(o_n), P(d_n), P(nr), P(fr), P(o_c), P(d_c), P(n_c), P(f_c),
           P(extra, allow_none=True), P(extra_c, allow_none=True), L.c_i32(0 if extra is None else extra.shape[1]), L.stream_ptr(), count=count)


def gather_rays_backward(idx, n, radius3, grads, vnorm, out, *, count=None):
    """nsb_gather_rays_backward: the adjoint of ray_test_aabb's normalisation, gather_rays and the view directions.  grads = (g_o, g_d,
    g_vd | None) [R, 3] in the caller's row order (row idx[j] of compacted ray j), vnorm [n] the compacted rays' clamped direction norms
    (None without g_vd), radius3 the box's host float[3] half-size -> out = (d_rays_o, d_rays_d) [R, 3], rows idx[:n] written (the caller
    zero-fills the others)"""
    (g_o, g_d, g_vd), (d_o, d_d), P = grads, out, L.ptr
    L.call(L.lib().nsb_gather_rays_backward, "gather_rays_backward", P(idx, "i64"), L.c_i64(n), radius3, P(g_o, "f32"), P(g_d, "f32"),
           P(g_vd, "f32", allow_none=True), P(vnorm, "f32", allow_none=True), P(d_o, "f32"), P(d_d, "f32"), L.stream_ptr(), count=count)


@torch.no_grad()
def merge_sorted_vals(dep_a, sdf_a, pack_infos_a, dep_b, sdf_b, *, n_out=None, count=None):
    """(dep_a, sdf_a) packs + rows of (dep_b, sdf_b)[P, nb] -> merged (dep, sdf | None, pack_infos); both sides sorted.  n_out: the
    length of the merged buffers (default: all samples)."""
    P, nb = dep_b.shape
    n = dep_a.shape[0] + P * nb if n_out is None else n_out
    dep_m = torch.empty(n, dtype=torch.float32, device=dep_a.device)
    sdf_m = torch.empty_like(dep_m) if sdf_a is not None else None
    pim = torch.empty_like(pack_infos_a)
    L.call(L.lib().nsb_merge_sorted_vals, "merge_sorted_vals", L.ptr(dep_a, "f32"), L.ptr(sdf_a, "f32", allow_none=True), L.ptr(pack_infos_a, "i64"),
           L.ptr(dep_b, "f32"), L.ptr(sdf_b, "f32", allow_none=True), L.c_i64(P), L.c_i32(nb), L.ptr(dep_m), L.ptr(sdf_m, allow_none=True),
           L.ptr(pim), L.stream_ptr(), count=count)
    return dep_m, sdf_m, pim


@torch.no_grad()
def assemble_boundary(coarse, ridx_hit, fine, run_len=None, *, want_mid=True, want_ridx=True, count=None):
    """coarse [R, nc] (sorted rows), fine [n_hit, nf] rows of rays ridx_hit, every row a concatenation of sorted runs of `run_len`
    samples (default: one run) -> (d1 [S], mid [S], ridx_all [S], pack_infos [R,2]); mid / ridx_all None unless wanted."""
    R, nc = coarse.shape
    n_hit, nf = (fine.shape if fine is not None else (0, 0))
    S, dev = R * nc + n_hit * nf, coarse.device
    d1 = torch.empty(S, dtype=torch.float32, device=dev)
    mid = torch.empty(S, dtype=torch.float32, device=dev) if want_mid else None
    ridx_all = torch.empty(S, dtype=torch.int64, device=dev) if want_ridx else None
    pi = torch.empty(R, 2, dtype=torch.int64, device=dev)
    run_len = [nf] if run_len is None else list(run_len)
    rl = (ctypes.c_int32 * len(run_len))(*run_len)
    L.call(L.lib().nsb_assemble_boundary, "assemble_boundary", L.ptr(coarse, "f32"), L.c_i64(R), L.c_i32(nc), L.ptr(ridx_hit, "i64", allow_none=True),
           L.c_i64(n_hit), L.ptr(fine, "f32", allow_none=True), L.c_i32(nf), rl, L.c_i32(len(run_len)), L.ptr(d1), L.ptr(mid, allow_none=True),
           L.ptr(ridx_all, "i64", allow_none=True), L.ptr(pi), L.stream_ptr(), count=count)
    return d1, mid, ridx_all, pi


def compact_samples(sel, pack_infos, first, steps, alpha, K, *, ridx_all=None, t_mid=None, d1=None, count=None):
    """nsb_compact_samples: the K (capacity) samples sel keeps -> (pidx, ridx, t, alpha) [K]; t and ridx from (ridx_all, t_mid), or, with
    d1, derived from the boundary depths and the packs"""
    dev = alpha.device
    pidx, ridx_c = torch.empty(K, dtype=torch.int64, device=dev), torch.empty(K, dtype=torch.int64, device=dev)
    t_c, alpha_c = torch.empty(K, dtype=torch.float32, device=dev), torch.empty(K, dtype=torch.float32, device=dev)
    P = L.ptr
    L.call(L.lib().nsb_compact_samples, "compact_samples", P(sel.view(torch.uint8), "u8"), P(pack_infos, "i64"), P(first, "i32"), P(steps, "i32"),
           L.c_i64(pack_infos.shape[0]), P(ridx_all, "i64", allow_none=True), P(t_mid, "f32", allow_none=True), P(d1, "f32", allow_none=True),
           P(alpha, "f32"), P(pidx), P(ridx_c), P(t_c), P(alpha_c), L.stream_ptr(), count=count)
    return pidx, ridx_c, t_c, alpha_c


def neus_alpha_compact(sdf, inv_s, pack_infos, ridx_all, t_mid, rays_inds, early_stop_eps=1e-4, alpha_thre=0.0):
    """neus_packed_sdf_to_alpha + packed_volume_render_compression + the gathers of the kept samples, 4 launches, 1 host read.
    -> None if nothing is kept, else dict(alpha [K] (differentiable wrt sdf, inv_s), ridx [K], t [K], pack_infos [Pu,2],
    nidx [Pu], rays_inds_hit [Pu], pidx [K])."""
    if not isinstance(inv_s, torch.Tensor):
        inv_s = torch.tensor(float(inv_s), device=sdf.device)
    alpha, sel, steps = _NeusAlpha.apply(sdf, inv_s, pack_infos, early_stop_eps, alpha_thre)
    with torch.no_grad():
        sc = scan_counts(steps, want_first=True, want_index=True, want_pack=True, src=rays_inds)
        K = sc["total"]
        if K == 0:
            return None
        pidx, ridx_c, t_c, alpha_c = compact_samples(sel, pack_infos, sc["first"], steps, alpha.detach(), K, ridx_all=ridx_all, t_mid=t_mid)
    alpha_k = _GatherUnique.apply(alpha, pidx, alpha_c) if alpha.requires_grad else alpha_c
    return dict(alpha=alpha_k, ridx=ridx_c, t=t_c, pack_infos=sc["pack"], nidx=sc["index"], rays_inds_hit=sc["src"], pidx=pidx)


_BITS_CACHE = {}


def pack_occ_bits(occ_grid):
    """the bool grid packed 32 cells / word (nsb_pack_occ_bits)"""
    cells = occ_grid.numel()
    words = torch.empty((cells + 31) // 32, dtype=torch.int32, device=occ_grid.device)
    L.check(L.lib().nsb_pack_occ_bits(L.ptr(occ_grid.contiguous().view(torch.uint8), "u8"), L.c_i64(cells), L.ptr(words), L.stream_ptr()), "pack_occ_bits")
    return words


@torch.no_grad()
def _occ_bits(occ_grid):
    """the packed grid, rebuilt only when the grid tensor changed"""
    key = (occ_grid.data_ptr(), occ_grid._version, tuple(occ_grid.shape))
    hit = _BITS_CACHE.get("k")
    if hit is None or hit[0] != key:
        hit = _BITS_CACHE["k"] = (key, pack_occ_bits(occ_grid), occ_grid)     # holds the grid: a freed + reallocated tensor cannot alias the key
    return hit[1]


def march_args(rays_o, rays_d, near, far, roi, occ_grid, step_size, max_step_size, dt_gamma, max_steps):
    """the leading arguments of nsb_ray_marching_listed, built once for both rounds of a march"""
    g = occ_grid.contiguous().view(torch.uint8)
    res = occ_grid.shape[-3:]
    return (L.c_i64(rays_o.shape[0]), L.ptr(rays_o, "f32", "rays_o"), L.ptr(rays_d, "f32", "rays_d"), L.ptr(near, "f32", "near"),
            L.ptr(far, "f32", "far"), L.ptr(roi, "f32", "roi"), None, L.c_i32(res[0]), L.c_i32(res[1]), L.c_i32(res[2]), L.ptr(g, "u8"),
            L.c_f32(step_size), L.c_f32(max_step_size), L.c_f32(dt_gamma), ctypes.c_uint32(int(max_steps)))


def march_listed(margs, bits, *, num_steps=None, info2=None, t_starts=None, ridx=None, ray_list=None, n_list=0, count=None):
    """one round of nsb_ray_marching_listed over margs (march_args): the first writes num_steps of every ray, the second the samples
    (t_starts, int32 ridx) of the n_list rays of ray_list at the offsets info2"""
    P = L.ptr
    L.call(L.lib().nsb_ray_marching_listed, "ray_marching", *margs, P(info2, allow_none=True), P(num_steps, allow_none=True),
           P(t_starts, allow_none=True), None, P(ridx, allow_none=True), None, None, P(ray_list, "i64", allow_none=True), L.c_i64(n_list),
           P(bits, allow_none=True), L.stream_ptr(), count=count)


@torch.no_grad()
def march_lean(occ_grid, rays_o, rays_d, near, far, *, step_size, max_steps, max_step_size=1e10, dt_gamma=0.0, roi=None):
    """occgrid_raymarch (graphics/raymarch.py) reduced to what the NeuS query consumes, without the per-sample temporaries:
    -> None if no ray hits an occupied voxel, else (ridx_hit [n_hit] i64, pack_infos [n_hit,2] i64, t_starts [M] f32, ridx [M] i64)."""
    R, dev = rays_o.shape[0], rays_o.device
    if roi is None:
        roi = torch.tensor([-1, -1, -1, 1, 1, 1], dtype=torch.float32, device=dev)
    args = march_args(rays_o, rays_d, near, far, roi, occ_grid, step_size, max_step_size, dt_gamma, max_steps)
    num_steps = torch.empty(R, dtype=torch.int32, device=dev)
    bits = _occ_bits(occ_grid) if occ_grid.numel() * 4 // 32 <= 96 * 1024 else None
    with L.KERNEL_TIMER.time("march", R):
        march_listed(args, bits, num_steps=num_steps)
    sc = scan_counts(num_steps, want_info2=True, want_index=True, want_pack=True)
    M = sc["total"]
    if M == 0:
        return None
    t_starts = torch.empty(M, dtype=torch.float32, device=dev)
    ridx = torch.empty(M, dtype=torch.int32, device=dev)
    with L.KERNEL_TIMER.time("march", R):
        march_listed(args, bits, info2=sc["info2"], t_starts=t_starts, ridx=ridx, ray_list=sc["index"], n_list=sc["n_nonzero"])
    return sc["index"], sc["pack"], t_starts, ridx.long()


class _Composite(torch.autograd.Function):
    @staticmethod
    def forward(ctx, alpha, t, rgb, nablas, pack_infos, normalize_depth, early_stop_eps, alpha_thre, ray_index, n_rays, count):
        a, tt = _f32c(alpha), _f32c(t)
        r = None if rgb is None else _f32c(rgb)
        nb = None if nablas is None else _f32c(nablas)
        P, dev = pack_infos.shape[0], a.device
        vw = torch.empty_like(a)
        n_out = P if ray_index is None else int(n_rays)
        cols = 2 + (3 if r is not None else 0) + (3 if nb is not None else 0)
        # whole-image buffers (rays without a pack stay 0): one allocation / zero-fill, four contiguous views
        buf = (torch.empty if ray_index is None else torch.zeros)(cols * n_out, device=dev)
        mask, depth = buf[:n_out], buf[n_out:2 * n_out]
        rgb_o = buf[2 * n_out:5 * n_out].view(n_out, 3) if r is not None else None
        o3 = 5 * n_out if r is not None else 2 * n_out
        nab_o = buf[o3:o3 + 3 * n_out].view(n_out, 3) if nb is not None else None
        L.call(L.lib().nsb_composite_forward, "composite_forward", L.ptr(a, "f32"), L.ptr(tt, "f32"), L.ptr(r, "f32", allow_none=True),
               L.ptr(nb, "f32", allow_none=True), L.ptr(pack_infos, "i64"), L.c_i64(P), L.c_f32(early_stop_eps), L.c_f32(alpha_thre),
               ctypes.c_int(1 if normalize_depth else 0), L.ptr(ray_index, "i64", allow_none=True), L.ptr(vw), L.ptr(mask), L.ptr(depth),
               L.ptr(rgb_o, allow_none=True), L.ptr(nab_o, allow_none=True), L.stream_ptr(), count=count)
        ctx.save_for_backward(a, tt, r, nb, vw, pack_infos, mask, depth, ray_index)
        ctx.cfg = (normalize_depth, early_stop_eps, alpha_thre, count)
        ctx.set_materialize_grads(False)
        empty = a.new_empty(0)
        return vw, mask, depth, (rgb_o if rgb_o is not None else empty), (nab_o if nab_o is not None else empty)

    @staticmethod
    def backward(ctx, g_vw, g_mask, g_depth, g_rgb, g_nab):
        a, tt, r, nb, vw, pack_infos, mask, depth, ray_index = ctx.saved_tensors
        normalize_depth, eps, thre, count = ctx.cfg
        P = pack_infos.shape[0]

        def opt(g, present=True):
            return None if (g is None or not present) else g.contiguous().float()
        g_vw, g_mask, g_depth = opt(g_vw), opt(g_mask), opt(g_depth)
        g_rgb, g_nab = opt(g_rgb, r is not None), opt(g_nab, nb is not None)
        d_alpha = torch.empty_like(a)
        d_rgb = torch.empty_like(r) if r is not None else None
        d_nab = torch.empty_like(nb) if nb is not None else None
        P_ = L.ptr
        L.call(L.lib().nsb_composite_backward, "composite_backward",
               P_(a, "f32"), P_(tt, "f32"), P_(r, allow_none=True), P_(nb, allow_none=True), P_(vw, "f32"), P_(pack_infos, "i64"), L.c_i64(P),
               L.c_f32(eps), L.c_f32(thre), ctypes.c_int(1 if normalize_depth else 0), P_(mask), P_(depth), P_(g_mask, allow_none=True),
               P_(g_depth, allow_none=True), P_(g_rgb, allow_none=True), P_(g_nab, allow_none=True), P_(g_vw, allow_none=True),
               P_(ray_index, "i64", allow_none=True), P_(d_alpha), P_(d_rgb, allow_none=True), P_(d_nab, allow_none=True), L.stream_ptr(), count=count)
        return d_alpha, None, d_rgb, d_nab, None, None, None, None, None, None, None


def composite(alpha, t, pack_infos, rgb=None, nablas=None, normalize_depth=True, early_stop_eps=1e-4, alpha_thre=0.0, ray_index=None,
              n_rays=None, count=None):
    """-> (vw [K], mask [P], depth [P], rgb [P,3] | None, normals [P,3] | None); differentiable wrt alpha, rgb, nablas.
    With `ray_index` [P] and `n_rays`, the per-ray outputs are whole-image buffers [n_rays(,3)] written at ray_index (zeros elsewhere)."""
    vw, mask, depth, rgb_o, nab_o = _Composite.apply(alpha, t, rgb, nablas, pack_infos, normalize_depth, early_stop_eps, alpha_thre,
                                                     ray_index, n_rays, count)
    return vw, mask, depth, (rgb_o if rgb is not None else None), (nab_o if nablas is not None else None)


@torch.no_grad()
def upsample_rays(meta, grid16, dec, ridx_hit, pack_infos, t_starts, rays_o, rays_d, inv_s_stages, num_fine, *, max_level, max_steps, use_estimate_alpha=False,
                  early_stop_eps=1e-4, alpha_thre=0.0, collect=None, count=None):
    """All up-sampling stages of the hit rays in ONE persistent kernel (csrc/ray_upsample.cu): sdf of the marched samples, then per stage
    cdf -> inverse-cdf samples -> sdf -> merge, the ray's samples in shared memory (long rays: a slice of a global scratch buffer).
    Replaces, with bit-identical results, the 11 launches `upsample_cdf / sample_cdf_uniform / fused_sdf_rays / merge_sorted_vals` make for
    three stages.  inv_s_stages[i] = upsample_inv_s * factor_i; num_fine: odd-ised counts.  max_steps None: no scratch, a ray that does not
    fit in shared memory is flagged in `overflow` instead.  -> (fine_all [n_hit, sum(num_fine)], overflow int32 [n_hit] (all zero unless
    a ray did not fit))."""
    n_hit, dev = ridx_hit.shape[0], t_starts.device
    n_stage = len(num_fine)
    us = [_quantiles(int(n), dev) for n in num_fine]
    fine_all = torch.empty(n_hit, int(sum(num_fine)), dtype=torch.float32, device=dev)
    overflow = torch.zeros(n_hit, dtype=torch.int32, device=dev)
    lib = L.lib()
    if max_steps is None:
        scratch, long_cap = None, 0
    else:
        long_cap = int(max_steps) + int(sum(num_fine[:-1])) + 64
        scratch = torch.empty(int(lib.nsb_upsample_rays_scratch_floats(L.c_i64(n_hit), L.c_i32(long_cap))), dtype=torch.float32, device=dev)
    nf = (ctypes.c_int32 * n_stage)(*[int(n) for n in num_fine])
    invs = (ctypes.c_float * n_stage)(*[float(v) for v in inv_s_stages])
    up = (ctypes.c_void_p * n_stage)(*[u.data_ptr() for u in us])
    with L.KERNEL_TIMER.time("ray_upsample", n_hit):
        L.call(lib.nsb_upsample_rays, "upsample_rays", meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(dec), L.ptr(rays_o, "f32"), L.ptr(rays_d, "f32"),
               L.ptr(t_starts, "f32"), L.ptr(pack_infos, "i64"), L.ptr(ridx_hit, "i64"), L.c_i64(n_hit), L.c_level(max_level), L.c_i32(n_stage), nf, invs, up,
               L.c_i32(1 if use_estimate_alpha else 0), L.c_f32(early_stop_eps), L.c_f32(alpha_thre), L.ptr(fine_all), L.ptr(overflow),
               L.ptr(scratch, allow_none=True), L.c_i32(long_cap), ctypes.byref(collect) if collect is not None else None, L.stream_ptr(), count=count,
               level=max_level)
    return fine_all, overflow


def upsample_persistent(surface, ridx_hit, pack_infos, t_starts, rays_o, rays_d, inv_s_stages, num_fine, use_estimate_alpha=False,
                        early_stop_eps=1e-4, alpha_thre=0.0, max_level=None):
    """`upsample_rays` of a LoTDSDF's fused query state without the scratch for long rays (they are flagged in `overflow`: 1 = this ray did
    not fit, its row is undefined)."""
    grid16, dec = surface._fused_state()
    return upsample_rays(surface.encoding.meta, grid16, dec, ridx_hit, pack_infos, t_starts, rays_o, rays_d, inv_s_stages, num_fine,
                         max_level=surface._ml(max_level), max_steps=None, use_estimate_alpha=use_estimate_alpha, early_stop_eps=early_stop_eps,
                         alpha_thre=alpha_thre)
