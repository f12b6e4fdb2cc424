"""Cost of the batch lookup in the LoTD table kernels: k_lotd_fwd (fp16 table, with dy_dx) and k_lotd_bwd_grid at 2 M points on the
16-level cfg3 table (auto_ngp_cfg([40, 150, 15], 32 Mi, 2^20)), unbatched against batched (four tables, unsorted batch_inds), timed
with CUDA events over alternating repeats.  The card's name and power limit are read in the same run.

    python profiles/lotd_batched_cost.py [--points 2097152] [--reps 50] [--out DIR]

Prints one JSON line (and writes it to DIR/lotd_batched_cost.json with --out)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=2 * 1024 * 1024)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from neuralsim_b200 import _lib as L
    from neuralsim_b200.bindings import _lotd
    from neuralsim_b200.fields.encoding import auto_ngp_cfg
    cfg = auto_ngp_cfg([40., 150., 15.], 32 * 2 ** 20, dim=3, n_feats=2, log2_hashmap_size=20, min_res=16, max_num_levels=16)
    m = _lotd.LoDMeta(3, cfg["lod_res"], cfg["lod_n_feats"], cfg["lod_types"], cfg["hashmap_size"])
    n, B, F = a.points, 4, m.n_encoded_dims
    g = torch.Generator("cuda").manual_seed(0)
    x = torch.rand(n, 3, device="cuda", generator=g).clamp_(1e-6, 1 - 1e-6)
    p = (torch.rand(B * m.n_params, device="cuda", generator=g) - 0.5).half()
    dLdy = (torch.randn(n, F, device="cuda", generator=g) * 0.1).half()
    inds = torch.randint(0, B, (n,), device="cuda", generator=g)
    y = torch.empty(n, F, dtype=torch.half, device="cuda")
    d = torch.empty(n, F * 3, device="cuda")
    acc = torch.zeros(B * m.n_params, device="cuda")
    lib = L.lib()
    batch = L.LotdBatchC(L.ptr(inds), None, 0)

    def fwd(bp):
        L.check(lib.nsb_lotd_fwd_batched(m.c_ref, L.ptr(x), L.ptr(p), 1, L.c_i64(n), L.c_i32(m.n_levels), bp, L.ptr(y), L.ptr(d),
                                         L.stream_ptr()), "fwd")

    def bwd(bp):
        L.check(lib.nsb_lotd_bwd_grid_batched(m.c_ref, L.ptr(dLdy), 1, L.ptr(x), L.c_i64(n), L.c_i32(m.n_levels), bp, L.c_f32(1.0),
                                              L.ptr(acc), L.stream_ptr()), "bwd_grid")

    variants = {"unbatched": L._NULL, "batched": ctypes.byref(batch)}
    for fn in (fwd, bwd):
        for bp in variants.values():
            for _ in range(5):
                fn(bp)
    torch.cuda.synchronize()
    times = {f"{k}_{v}": [] for k in ("fwd", "bwd_grid") for v in variants}
    for _ in range(a.reps):                        # alternate the variants so that clock drift hits both alike
        for name, fn in (("fwd", fwd), ("bwd_grid", bwd)):
            for v, bp in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(bp)
                e1.record()
                e1.synchronize()
                times[f"{name}_{v}"].append(e0.elapsed_time(e1))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = dict(points=n, tables=B, levels=m.n_levels, reps=a.reps, device=torch.cuda.get_device_name(0),
               nvidia_smi=smi[0] if smi else None,
               median_ms={k: float(np.median(v)) for k, v in times.items()},
               p10_p90_ms={k: [float(np.percentile(v, 10)), float(np.percentile(v, 90))] for k, v in times.items()})
    res["batched_over_unbatched"] = {k: res["median_ms"][f"{k}_batched"] / res["median_ms"][f"{k}_unbatched"] for k in ("fwd", "bwd_grid")}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lotd_batched_cost.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
