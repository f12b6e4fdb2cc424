"""Outputs of the reference project's own CUDA kernels on the inputs of the parity tests, kept under tests/golden/ so that
the comparisons run anywhere.  The reference kernels are compiled into oracle/_ref by oracle/build_ref.py; with
NSB_RECORD_REF=<dir> set (on a GPU machine where oracle/_ref is built) the tests call them and write ref_<name>.npz to <dir>.

A bit-exact comparison stores the SHA-256 digest of the reference output (shape, dtype and bytes); a comparison with a
tolerance stores the values, or a fixed part of them where the whole array would be too large to keep."""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
RECORD = os.environ.get("NSB_RECORD_REF")


def digest(t):
    t = t.detach().contiguous().cpu()
    return hashlib.sha256(repr((tuple(t.shape), str(t.dtype))).encode() + t.numpy().tobytes()).hexdigest()


class Golden:
    def __init__(self, name, module=None):
        """name: of the golden file (ref_<name>.npz); module: the reference extension in oracle/_ref (default: name)"""
        self.name, self.rec = name, {}
        if RECORD:
            sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
            import build_ref
            self.ref = build_ref.load(module or name)
            assert self.ref is not None, f"oracle/_ref/{module or name} is not built"
        else:
            self.ref = None
            self.rec = dict(np.load(os.path.join(HERE, "golden", f"ref_{name}.npz")))

    def value(self, key, fn):
        """fn(reference module) -> tensor; returns the reference value as a CPU tensor"""
        if RECORD:
            self.rec[key] = fn(self.ref).detach().contiguous().cpu().numpy()
        return torch.from_numpy(self.rec[key])

    def equal(self, key, ours, fn):
        """asserts that `ours` is bit for bit the reference's fn(reference module)"""
        if RECORD:
            self.rec[key] = np.array(digest(fn(self.ref)))
        assert digest(ours) == str(self.rec[key]), key

    def save(self):
        if RECORD:
            os.makedirs(RECORD, exist_ok=True)
            np.savez_compressed(os.path.join(RECORD, f"ref_{self.name}.npz"), **self.rec)
