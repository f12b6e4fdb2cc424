"""How many table-gradient reductions do the two SDF backward kernels issue in the bench step, and how many would merging the runs of
same-cell lanes on EVERY level save?  One kernel-by-kernel StaticFrame step of the bench workload (cfg2: one 800x600 frame, fwd+bwd) on
the GPU; the census itself is counted from the step's own samples, in the lane order the kernels see them:
  k_color_sdf_bwd  the kept samples (the colour query's points, ray-ordered), every lane active
  k_sdf_bwd_tc     the sdf-backward list (each kept sample and the boundary sample after it), a lane active when its d_sdf != 0
A warp of 32 consecutive work items issues, per level, one 8-corner reduction per active run head (warp_merge_updates, csrc/
lotd_device.cuh); with more than 24 run heads (inactive lanes count as heads) every active lane issues its own.
  old rule: runs are merged only on levels with <= 1024 cells per axis; on the others every active lane issues
  new rule: runs are merged on every level
    python profiles/scatter_census.py
Prints a table per kernel (8-reduction issues per level, old / new) and one JSON line with the totals, the share saved and the GPU name
and power limit."""
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import bench  # noqa: E402
from bwd_kernels import gpu_info  # noqa: E402
from neuralsim_b200.graphics import neus_static  # noqa: E402
from neuralsim_b200.graphics.neus_static import CNT_SLOTS, StaticFrame  # noqa: E402

MAX_HEADS = 24                      # warp_merge_updates: more run heads than this -> every lane issues its own


def census(x, active, res):
    """x [N, 3] network-space points in lane order, active [N] bool, res [L][3] -> per level (issues old rule, issues new rule, warps
    with > MAX_HEADS heads, warps) as python ints"""
    n = x.shape[0]
    W = -(-n // 32) * 32
    dev = x.device
    xp = torch.zeros(W, 3, dtype=torch.float32, device=dev)
    xp[:n] = x
    act = torch.zeros(W, dtype=torch.bool, device=dev)
    act[:n] = active
    xs = (xp * 0.5 + 0.5).clamp(1.0e-6, 1.0 - 1.0e-6)                   # to_table_space (x * 0.5 is exact: one rounding, as the fma)
    prev_act = torch.zeros_like(act)
    prev_act[1:] = act[:-1]
    prev_act = prev_act.view(-1, 32)
    prev_act[:, 0] = False
    act32 = act.view(-1, 32)
    out = []
    for r in res:
        sc = torch.tensor([float(v - 2) for v in r], dtype=torch.float64, device=dev)
        v = (xs.double() * sc + 0.5).float()                             # fma(xs, scale, 0.5): exact product, one rounding to fp32
        cell = torch.floor(v).to(torch.int64).view(-1, 32, 3)
        differs = torch.ones(cell.shape[:2], dtype=torch.bool, device=dev)
        differs[:, 1:] = (cell[:, 1:] != cell[:, :-1]).any(-1)
        head = ~act32 | ~prev_act | differs
        heads = head.sum(1)
        n_act = act32.sum(1)
        n_act_heads = (act32 & head).sum(1)
        merged = torch.where(heads > MAX_HEADS, n_act, n_act_heads)
        mergeable = all(v <= 1024 for v in r)
        old = int((merged if mergeable else n_act).sum())
        out.append((old, int(merged.sum()), int((heads > MAX_HEADS).sum()), heads.shape[0]))
    return out


def report(name, rows, res):
    print(f"{name}: 8-reduction issues per level (old rule -> new rule; warps with > {MAX_HEADS} heads)")
    for l, ((old, new, full, warps), r) in enumerate(zip(rows, res)):
        print(f"  L{l:<2d} res {r[0]:5d}  {old:10d} -> {new:10d}  ({100.0 * (old - new) / max(old, 1):5.1f} % saved; {full}/{warps} warps unmerged)")
    old, new = sum(r[0] for r in rows), sum(r[1] for r in rows)
    print(f"  total {old} -> {new}: {100.0 * (old - new) / max(old, 1):.1f} % of the kernel's reductions saved", flush=True)
    return dict(issues_old=old, issues_new=new, saved=round((old - new) / max(old, 1), 4),
                per_level=[dict(level=l, old=a, new=b, warps_unmerged=c, warps=w) for l, (a, b, c, w) in enumerate(rows)])


def main():
    dev = torch.device("cuda:0")
    model = bench.build_model(dev).train()
    flat, _ = bench.flat_grad_views(model)
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(0, bench.N_VIEWS))
    o, d = o.to(dev), d.to(dev)
    seen = {}
    sdf_bwd = neus_static.sdf_bwd

    def sdf_bwd_seen(meta, grid16, dec, d_sdf, n, max_level, grads, **kw):
        seen.update(d_sdf=d_sdf, rays=kw["rays"], keep=kw["keep"])
        return sdf_bwd(meta, grid16, dec, d_sdf, n, max_level, grads, **kw)

    neus_static.sdf_bwd = sdf_bwd_seen
    frame = StaticFrame(model, o.shape[0], loss_fn=bench.loss_of, near=0.01, use_graph=False, pre_hook=flat.zero_)
    for _ in range(3):
        frame.step(o, d, None)
    torch.cuda.synchronize()
    c = frame.counts()
    assert c["overflow"] == 0, c
    meta = model.implicit_surface.encoding.meta
    ml = model.implicit_surface._ml(model.max_level)
    res = [r for l, r in enumerate(meta.level_res_multidim) if ml < 0 or l <= ml]
    K, nz = c["kept"], c["nonzero"]
    xk = frame.buffers["net_x"][:K].detach()
    col = census(xk, torch.ones(K, dtype=torch.bool, device=dev), res)
    keep = seen["keep"][:nz]
    ro, rd, ray, t = seen["rays"]
    r = ray[keep]
    xb = torch.addcmul(ro[r], rd[r], t[keep].unsqueeze(-1))            # fma(d, t, o) per component
    sdf = census(xb, seen["d_sdf"][keep] != 0, res)
    line = dict(kept=K, sdf_bwd_list=nz, k_color_sdf_bwd=report("k_color_sdf_bwd (kept samples)", col, res),
                k_sdf_bwd_tc=report("k_sdf_bwd_tc (sdf-backward list)", sdf, res))
    old = line["k_color_sdf_bwd"]["issues_old"] + line["k_sdf_bwd_tc"]["issues_old"]
    new = line["k_color_sdf_bwd"]["issues_new"] + line["k_sdf_bwd_tc"]["issues_new"]
    line.update(issues_old=old, issues_new=new, saved=round((old - new) / max(old, 1), 4), **gpu_info())
    print(f"both kernels: {old} -> {new} 8-reduction issues per step, {100.0 * (old - new) / max(old, 1):.1f} % saved")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
