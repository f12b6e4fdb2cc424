"""Host-side logic that needs no GPU: bench.py helpers, the renderer's lazy image buffers, profile summarisers."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_effective_cpus_and_disabled_sampler():
    import bench
    n = bench.effective_cpus()
    assert 1 <= n <= (os.cpu_count() or 1)
    cs = bench.ClockSampler(0, 0)                     # period 0 = diagnostics mode: never forks, never samples
    with cs:
        cs.sample()
    assert cs.summary()["sm_mhz"] is None and cs.summary()["reasons"] == ["no sampler"]


def test_lazy_rendered_buffers():
    from neuralsim_b200.renderer import _LazyZeros
    r = _LazyZeros(5, "cpu", with_rgb=True, with_normal=False)
    assert "rgb_volume" in r and "normals_volume" not in r and len(dict(r)) == 0        # nothing allocated yet
    assert r["mask_volume"].shape == (5,) and float(r["mask_volume"].abs().sum()) == 0
    r["depth_volume"] = torch.ones(5)                 # a consumer may replace a buffer wholesale
    out = r.materialise()
    assert sorted(out) == ["depth_volume", "mask_volume", "rgb_volume"] and out["rgb_volume"].shape == (5, 3)
    assert float(out["depth_volume"].sum()) == 5.0
    try:
        r["normals_volume"]
        raise AssertionError("a buffer that was not requested must not appear")
    except KeyError:
        pass


def _h100_line():
    import json
    return json.loads(open(os.path.join(ROOT, "profiles", "h100_bench.json")).read().strip().splitlines()[-1])


def test_bench_line_files_are_valid_json():
    d = _h100_line()
    for k in ("metric", "value", "unit", "n_gpus", "ms_per_step", "higher_is_better", "scaling", "e2e", "gpu_launches", "roofline", "config"):
        assert k in d, k
    assert d["gpu_launches"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0


def test_march_onepass_gate_and_final_bench_line():
    """the recorded one-pass march is a small-batch path (record <= 64 MB unless forced); the stored H100 bench line of the default
    invocation keeps the bench line's keys"""
    from neuralsim_b200.graphics import neus_static as NS
    old = NS.MARCH_ONEPASS
    try:
        NS.MARCH_ONEPASS = "auto"
        assert NS.march_onepass(4096, 1024) and NS.march_onepass(16384, 1024) and not NS.march_onepass(480000, 1024)
        NS.MARCH_ONEPASS = "0"
        assert not NS.march_onepass(16, 16)
        NS.MARCH_ONEPASS = "1"
        assert NS.march_onepass(480000, 1024)
    finally:
        NS.MARCH_ONEPASS = old
    d = _h100_line()
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "dtype", "data", "config", "e2e", "gpu_launches",
              "roofline", "cpu_baseline", "clocks", "median", "reference_cuda", "vs_reference_cuda", "parity_vs_reference_kernels"):
        assert k in d, k
    assert d["config"]["workload"] == "cfg2" and d["e2e"]["d2h_bytes_per_step"] > 15_000_000 and d["e2e"]["value"] < d["value"]
    assert len(d["step_ms"]["resident"]) == d["steps"]
    r = d["roofline"]
    assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert abs(d["vs_reference_cuda"]["value_ratio"] - d["value"] / d["reference_cuda"]["value"]) < 1e-9
    assert all(d["parity_vs_reference_kernels"][k]["rel_l2"] <= 1e-4 for k in ("rgb_volume", "depth_volume", "normals_volume"))
    assert d["step_ms"]["resident_stats"]["max"] / d["step_ms"]["resident_stats"]["median"] <= 1.15
