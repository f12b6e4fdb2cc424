"""Mesh extraction at N = 512 (neuralsim_b200.graphics.trianglemesh.extract_mesh, the call of neuralsim's code_single/tools/extract_mesh.py):
    python profiles/mesh_extract.py [--N 512] [--chunk 8388608] [--out DIR]

Workloads:
  cfg3_17  the full-size cfg3 street model (bench_cfg3.build_model: 40 x 150 x 15 m, 32 Mi-parameter table) with 17 levels (the shipped
           table: the generic encoding -> decoder path), whole box: a 1365 x 5120 x 512 lattice (3.58 G points)
  cfg3_16  the same with 16 levels (the fused k_fused_sdf_tc query)
  sphere   the CFG sphere model (tests/util.make_pair) on [-1, 1]^3: 512^3
Each is warmed up once at N = 64, then timed once with colours (the radiance net at v = -normal, zero appearance code) and the PLY file
written to a temporary directory.  Prints one JSON line per workload: seconds of lattice + SDF query, marching cubes, colour (+ the
scale / offset / transform step, none here), PLY write, and in all; vertex and face counts; torch.cuda.max_memory_allocated; and the GPU
name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the numbers stand without it, but say why it is missing
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def workloads(dev):
    import bench_cfg3 as C
    from util import make_pair

    def cfg3(levels):
        def make():
            m = C.build_model(dev, max_num_levels=levels).eval()
            assert m.implicit_surface.encoding.meta.n_levels == levels and m.implicit_surface._fusable() == (levels == 16)
            return m, np.array(C.AABB[0]), np.array(C.AABB[1])
        return make

    def sphere():
        _, m = make_pair(dev)
        return m.eval(), np.array([-1., -1., -1.]), np.array([1., 1., 1.])
    return dict(cfg3_17=cfg3(17), cfg3_16=cfg3(16), sphere=sphere)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=512)
    ap.add_argument("--chunk", type=int, default=8 * 2 ** 20)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    args = ap.parse_args()
    from neuralsim_b200.graphics.trianglemesh import extract_mesh
    dev = torch.device("cuda:0")
    info = gpu_info()
    for name, make in workloads(dev).items():
        if args.only and name not in args.only.split(","):
            continue
        model, bmin, bmax = make()
        q = lambda x: model.forward_sdf(model.space.normalize_coords(x))["sdf"]
        n_h = model.implicit_surface.encoding.out_features
        n_appear = model.radiance_net.blocks.layers[0].weight.shape[1] - (3 + 16 + 3 + n_h)        # inputs [x, SH4(v), n, h, h_appear]
        h0 = torch.zeros(1, n_appear, device=dev)
        col = lambda x, v: model.forward(model.space.normalize_coords(x), v=v, h_appear=h0, with_normal=True)["rgb"].float()
        with tempfile.TemporaryDirectory() as tmp:
            kw = dict(query_color_fn=col, include_color=True, show_progress=False, bmin=bmin, bmax=bmax, chunk=args.chunk, device=dev)
            extract_mesh(q, filepath=os.path.join(tmp, "warm.ply"), N=64, **kw)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            out = extract_mesh(q, filepath=os.path.join(tmp, "mesh.ply"), N=args.N, **kw)
            ply_bytes = os.path.getsize(os.path.join(tmp, "mesh.ply"))
        n = [int(v) for v in (((bmax - bmin) / (bmax - bmin).min()) * args.N).astype(np.int32)]
        print(json.dumps(dict(workload=name, lattice=n, points=int(np.prod(n)), chunk=args.chunk, verts=int(out["verts"].shape[0]),
                              faces=int(out["faces"].shape[0]), seconds={k: round(v, 4) for k, v in out["timing"].items()},
                              max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), ply_bytes=ply_bytes, **info)),
              flush=True)
        del model, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
