"""Every output of nsb_fused_color_fwd from this checkout against another checkout (--parent ROOT, its library built), bit for bit.

Inputs: the kept samples of the bench frame (bench.py: cfg2 model, view 0, 800x600 rays, host-sized render: the samples and rays the colour
query receives), and their first 1, 127, 128, 129 and 67 k samples (the last a size at which every persistent CTA of k_color_fwd loops),
that size with max_level 5, and that capacity with a device count below it.  For each, both instantiations: k_color_fwd<true> (sdf,
nablas, rgb, x, the saved Z / X / Y1 / Y2 tiles) and k_color_fwd<false> (sdf, nablas, x, Z and X tiles).

The inputs are captured once (a process with this checkout) and each checkout runs in its own process, writing its outputs as .npy into a
temporary directory (about 2.5 GB per checkout on the bench frame); the directories are compared file by file and removed.  Prints one JSON
line per case and a summary line with the GPU name, power limit and SM clock.
    python profiles/color_fwd_bit_equal.py --parent ROOT [--keep DIR]"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cases(n_kept, sms):
    loop = (2 * sms * 2 + 1) * 128 - 51
    out = [("frame", n_kept, None, None)] + [(f"n{n}", n, None, None) for n in (1, 127, 128, 129, loop)]
    out += [(f"n{loop}_ml5", loop, 5, None), (f"n{loop}_count", loop, None, loop - sms * 128 - 37)]
    return [c for c in out if c[1] <= n_kept]


def capture(args):
    """the bench model's state and the arguments of the colour query of the bench frame's host-sized render"""
    sys.path.insert(0, ROOT)
    import importlib
    import torch
    import bench
    FC = importlib.import_module("neuralsim_b200.fields.fused_color")
    from neuralsim_b200.renderer import SingleVolumeRenderer
    dev = torch.device("cuda", 0)
    model = bench.build_model(dev).train()
    o, d = bench.pinhole_rays(bench.H, bench.W, bench.orbit(0, bench.N_VIEWS))
    rec = []
    orig = FC._FusedColor.forward

    def spy(ctx, q, ridx, t, view_dirs, h_appear, keep, *params):
        rec.append(dict(ridx=ridx, t=t, view_dirs=view_dirs, h_appear=h_appear, rays_o=q.rays_o, rays_d=q.rays_d))
        return orig(ctx, q, ridx, t, view_dirs, h_appear, keep, *params)
    FC._FusedColor.forward = staticmethod(spy)
    with torch.no_grad():
        SingleVolumeRenderer(dict(near=0.01)).train().render(model, o.to(dev), d.to(dev), rays_h_appear=torch.zeros(o.shape[0], 4, device=dev))
    assert len(rec) == 1 and model.max_level is None, len(rec)
    r = rec[0]
    torch.save(dict(state=model.state_dict(), **{k: v.cpu() for k, v in r.items()}), os.path.join(args.dir, "inputs.pt"))
    print(json.dumps(dict(kept=int(r["t"].numel()), sms=torch.cuda.get_device_properties(0).multi_processor_count)), flush=True)


def dump(args):
    """this process's library: every output of nsb_fused_color_fwd for every case and both instantiations -> args.dir/<case>_<inst>_<key>.npy"""
    sys.path.insert(0, args.root)
    import torch
    import bench
    from neuralsim_b200 import _lib as L
    dev = torch.device("cuda", 0)
    inp = torch.load(os.path.join(os.path.dirname(args.dir.rstrip("/")), "inputs.pt"))
    model = bench.build_model(dev).train()
    model.load_state_dict(inp["state"])
    s = model.implicit_surface
    lib = L.lib()
    g = {k: inp[k].to(dev).contiguous() for k in ("ridx", "t", "view_dirs", "h_appear", "rays_o", "rays_d")}
    os.makedirs(args.dir, exist_ok=True)
    for name, n, max_level, count in _cases(g["t"].numel(), torch.cuda.get_device_properties(0).multi_processor_count):
        for rad in (True, False):
            grid16, net, _held = model._fused_color_state() if rad else model._fused_geometry_state()
            nan = float("nan")
            out = dict(sdf=torch.full((n,), nan, device=dev), nablas=torch.full((n, 3), nan, device=dev), x=torch.full((n, 3), nan, device=dev))
            if rad:
                out["rgb"] = torch.full((n, 3), nan, device=dev)
            tb = int(lib.nsb_color_tile_bytes(L.c_i64(n)))
            names = ("Z", "X", "Y1", "Y2") if rad else ("Z", "X")
            for k in names:
                out[k] = torch.full((tb,), 0xA5, dtype=torch.uint8, device=dev)      # bytes the kernel does not write stay recognisable
            ap = [L.ptr(out[k]) if k in out else None for k in ("Z", "X", "Y1", "Y2")]
            cnt = torch.tensor([count if count is not None else n], dtype=torch.int64, device=dev)
            if count is not None:
                lib.nsb_bind_device_counts(ctypes.c_void_p(cnt.data_ptr()), ctypes.c_void_p(0))
            try:
                rc = lib.nsb_fused_color_fwd(s.encoding.meta.c_ref, L.ptr(grid16, "f16"), ctypes.byref(net), None, L.ptr(g["rays_o"], "f32"),
                                             L.ptr(g["rays_d"], "f32"), L.ptr(g["ridx"][:n], "i64"), L.ptr(g["t"][:n], "f32"),
                                             L.ptr(g["view_dirs"], "f32") if rad else None, L.ptr(g["h_appear"], "f32") if rad else None,
                                             L.c_i64(n), L.c_i32(s._ml(max_level)), L.ptr(out["sdf"]), L.ptr(out["nablas"]),
                                             L.ptr(out["rgb"]) if rad else None, L.ptr(out["x"]), *ap, None, L.stream_ptr())
            finally:
                if count is not None:
                    lib.nsb_bind_device_counts(ctypes.c_void_p(0), ctypes.c_void_p(0))
            L.check(rc, "fused_color_fwd")
            torch.cuda.synchronize()
            for k, v in out.items():
                np.save(os.path.join(args.dir, f"{name}_{'true' if rad else 'false'}_{k}.npy"), v.cpu().numpy())
            del out
    print(json.dumps(dict(dumped=args.root)), flush=True)


def _run(cmd):
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{p.stdout[-4000:]}\n{p.stderr[-4000:]}")
    return [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None)
    ap.add_argument("--keep", default=None, help="keep the inputs and both checkouts' outputs under this directory")
    ap.add_argument("--capture", action="store_true")
    ap.add_argument("--dump", action="store_true")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    if args.capture:
        return capture(args)
    if args.dump:
        return dump(args)
    if not args.parent:
        raise SystemExit("color_fwd_bit_equal.py: --parent ROOT is required")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    base = args.keep or tempfile.mkdtemp(prefix="nsb_color_fwd_")
    os.makedirs(base, exist_ok=True)
    me = os.path.abspath(__file__)
    try:
        info = _run([sys.executable, me, "--capture", "--dir", base])[0]
        dirs = {}
        for name, root in (("built", ROOT), ("parent", os.path.abspath(args.parent))):
            dirs[name] = os.path.join(base, name)
            _run([sys.executable, me, "--dump", "--root", root, "--dir", dirs[name]])
        files = sorted(os.listdir(dirs["built"]))
        assert files == sorted(os.listdir(dirs["parent"])) and files, "the two checkouts wrote different files"
        per_case, all_equal = {}, True
        for f in files:
            a, b = np.load(os.path.join(dirs["built"], f)), np.load(os.path.join(dirs["parent"], f))
            eq = a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
            case = f.rsplit("_", 1)[0]
            per_case.setdefault(case, {})[f.rsplit("_", 1)[1][:-4]] = eq
            all_equal &= eq
        for case, r in per_case.items():
            print(json.dumps(dict(case=case, bit_equal=r)), flush=True)
        print(json.dumps(dict(all_bit_equal=bool(all_equal), files=len(files), **info, gpu=q.stdout.strip())), flush=True)
    finally:
        if not args.keep:
            shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
