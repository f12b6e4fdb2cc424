"""Parity AT THE BENCHMARK'S OWN SIZE (BASELINE.json: "PSNR vs ref"; north_star: rgb / depth / normals within 1e-4 relative L2 on identical rays
and weights): the 800x600 frame of bench.py rendered by our kernels (host-sized fused path AND the static / graph path) against the render of the
REFERENCE'S OWN KERNELS (oracle/_ref: `_lotd`, `_pack_ops`, `_occ_grid`, `_shencoder` compiled by oracle/build_ref.py, driven op by op).  The
reference renders are stored for a fixed sample of pixels in tests/golden/ref_frames.npz; NSB_RECORD_REF=<dir> re-records them where oracle/_ref
is built (the reference arm runs in a child process: it patches module-level back ends).  Also: 4096 random rays (MODE-1 traversal, the
training batch)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
KEYS = ("rgb_volume", "depth_volume", "normals_volume", "mask_volume")
RECORD = os.environ.get("NSB_RECORD_REF")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_frames.npz")
N_PIX = 8192                                  # pixels of a frame kept: a fixed seeded sample

CHILD = r'''
import sys, torch
sys.path.insert(0, %(root)r)
import bench
assert bench.use_reference_cuda_kernels(), "oracle/_ref is not built"
from neuralsim_b200.renderer import SingleVolumeRenderer
dev = torch.device("cuda:0")
model = bench.build_model(dev, collect_samples=%(collect)r)
model.train(%(train)r)
o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(%(view)d, 8))
if %(random)r:
    sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(11))[:4096]
    o, d = o[sel].contiguous(), d[sel].contiguous()
r = SingleVolumeRenderer(dict(near=0.01)).train(%(train)r)
with torch.no_grad():
    out = r.render(model, o.to(dev), d.to(dev), rays_h_appear=torch.zeros(o.shape[0], 4, device=dev))["rendered"]
torch.save({k: v.cpu() for k, v in out.items()}, %(path)r)
'''


def _pixels(n):
    return torch.randperm(n, generator=torch.Generator().manual_seed(3))[:N_PIX].sort().values if n > N_PIX else torch.arange(n)


def _reference_render(tmp_path, view, train, random, collect=False):
    """the reference kernels' render at the pixels _pixels(number of rays)"""
    tag = f"view{view}_{int(train)}_{int(random)}"
    if RECORD:
        path = str(tmp_path / f"ref_{tag}.pt")
        code = CHILD % dict(root=ROOT, view=view, train=train, random=random, collect=collect, path=path)
        subprocess.run([sys.executable, "-c", code], check=True, timeout=600)
        full = torch.load(path)
        sel = _pixels(full[KEYS[0]].shape[0])
        rec = dict(np.load(os.path.join(RECORD, "ref_frames.npz"))) if os.path.exists(os.path.join(RECORD, "ref_frames.npz")) else {}
        rec.update({f"{tag}.{k}": full[k][sel].numpy() for k in KEYS})
        os.makedirs(RECORD, exist_ok=True)
        np.savez_compressed(os.path.join(RECORD, "ref_frames.npz"), **rec)
    gold = np.load(GOLDEN) if not RECORD else np.load(os.path.join(RECORD, "ref_frames.npz"))
    return {k: torch.from_numpy(gold[f"{tag}.{k}"]) for k in KEYS}


def _report(tag, got, ref):
    res = {}
    for k in KEYS:
        x, y = got[k].detach().double().cpu(), ref[k].double()
        mse = float((x - y).square().mean())
        res[k] = dict(rel_l2=float((x - y).norm() / y.norm().clamp_min(1e-30)), psnr_db=(None if mse == 0 else -10.0 * float(torch.log10(torch.tensor(mse)))))
    print(tag, json.dumps(res))
    return res


@pytest.mark.parametrize("view,train", [(0, False), (3, True)])
def test_800x600_frame_vs_the_reference_kernels(cuda, tmp_path, view, train):
    import bench
    from neuralsim_b200.renderer import SingleVolumeRenderer
    from neuralsim_b200.graphics.neus_static import StaticFrame
    ref = _reference_render(tmp_path, view, train, False)
    sel = _pixels(bench.H * bench.W)
    model = bench.build_model(cuda).train(train)
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(view, 8))
    o, d, ha = o.to(cuda), d.to(cuda), torch.zeros(bench.H * bench.W, 4, device=cuda)
    with torch.no_grad():
        got = SingleVolumeRenderer(dict(near=0.01)).train(train).render(model, o, d, rays_h_appear=ha)["rendered"]
        res = _report(f"frame view {view} {'train' if train else 'eval'} (host-sized fused path, {N_PIX} pixels)", {k: got[k][sel.to(cuda)] for k in KEYS}, ref)
        for k in ("rgb_volume", "depth_volume", "normals_volume"):
            assert res[k]["rel_l2"] <= 1e-4, (k, res[k])
        assert res["rgb_volume"]["psnr_db"] is None or res["rgb_volume"]["psnr_db"] >= 80.0
        frame = StaticFrame(model, o.shape[0], near=0.01)          # the graph step renders the same images bit for bit
        frame.step(o, d, ha)
        assert frame.counts()["overflow"] == 0
        for k in KEYS:
            assert torch.equal(frame.rendered[k], got[k]), k


def test_4096_random_rays_vs_the_reference_kernels(cuda, tmp_path):
    import bench
    from neuralsim_b200.renderer import SingleVolumeRenderer
    ref = _reference_render(tmp_path, 5, True, True, collect=True)
    model = bench.build_model(cuda, collect_samples=True).train()
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(5, 8))
    sel = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(11))[:4096]
    o, d = o[sel].contiguous().to(cuda), d[sel].contiguous().to(cuda)
    with torch.no_grad():
        got = SingleVolumeRenderer(dict(near=0.01)).train().render(model, o, d, rays_h_appear=torch.zeros(4096, 4, device=cuda))["rendered"]
    res = _report("4096 random rays, training mode, sample collection on", got, ref)
    for k in ("rgb_volume", "depth_volume", "normals_volume"):
        assert res[k]["rel_l2"] <= 1e-4, (k, res[k])
    assert float(model.accel.occ._occ_val_grid_pcl.sum()) > 0          # the in-kernel collection ran
