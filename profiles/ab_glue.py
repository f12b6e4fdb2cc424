"""A/B of the graph-captured step's march on one GPU, one process, same model and poses (not a bench value; bench.py is):
   onepass     0 = two-round march, 1 = march once recording the samples per ray + copy (auto: only when the record fits 64 MB)
(r02j: the first version of this script captured its second frame with all-zero input rays and hung in the march until its timeout; only the
first configuration of each run was recorded.  Fixed below.)
Usage: python profiles/ab_glue.py [--rays 480000 | --rays 4096 --random-rays] [--steps 20] [--rounds 2]"""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=bench.H * bench.W)
    ap.add_argument("--random-rays", action="store_true")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    from neuralsim_b200.graphics import neus_static as NS
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    model = bench.build_model(dev).train()
    flat, _ = bench.flat_grad_views(model)
    views = []
    for k in range(5):
        o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(k, bench.N_VIEWS))
        if args.random_rays:
            sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(1000 + k))[:args.rays]
            o, d = o[sel], d[sel]
        else:
            o, d = o[:args.rays], d[:args.rays]
        views.append((o.contiguous().to(dev), d.contiguous().to(dev)))
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    caps = {}

    def run(onepass):
        NS.MARCH_ONEPASS = onepass
        fr = NS.StaticFrame(model, args.rays, loss_fn=bench.loss_of, near=0.01, pre_hook=flat.zero_, **caps)
        if not caps:
            for o, d in views:
                fr.rays_o.copy_(o); fr.rays_d.copy_(d)
                fr._size()
            caps.update(march_cap=fr.march_cap, kept_cap=fr.kept_cap, coherent=fr.coherent)
        fr.rays_o.copy_(views[0][0]); fr.rays_d.copy_(views[0][1])     # the capture's warm-up must see real rays (all-zero directions march forever)
        fr.capture()
        for i in range(args.warmup):
            fr.step(*views[i % len(views)])
        torch.cuda.synchronize()
        evs = []
        for i in range(args.steps):
            flush.fill_(i & 0xff)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fr.step(*views[i % len(views)]); b.record()
            evs.append((a, b))
        torch.cuda.synchronize()
        ts = sorted(a.elapsed_time(b) for a, b in evs)
        assert fr.counts()["overflow"] == 0
        chk = float(fr.rendered["rgb_volume"].detach().double().sum()), float(fr.rendered["depth_volume"].detach().double().sum())
        del fr
        gc.collect()
        torch.cuda.empty_cache()
        return dict(onepass=onepass, mean=sum(ts) / len(ts), median=ts[len(ts) // 2], min=ts[0], max=ts[-1], checksum=chk)

    for r in range(args.rounds):
        for onepass in ("0", "1"):
            print(json.dumps(dict(rays=args.rays, round=r, **run(onepass))), flush=True)


if __name__ == "__main__":
    main()
