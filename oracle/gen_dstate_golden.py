"""Golden vectors of the selective scan at 32 and 64 states from the REFERENCE's own `selective_scan_ref` (needs the reference
checkout).  TEST INFRASTRUCTURE, like oracle/gen_golden.py, whose reference loader it uses: forward outputs, the last state and
every input gradient of the cases in tests/dstate_cases.py, written to tests/golden/scan_dstate*.npz.

Usage:  python oracle/gen_dstate_golden.py
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen_golden():
    spec = importlib.util.spec_from_file_location("gen_golden", os.path.join(HERE, "gen_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    gg = _gen_golden()
    sys.path.insert(0, os.path.dirname(gg.OUT))
    from dstate_cases import DSTATE_CASES
    from golden_inputs import scan_inputs
    ssi, _ = gg.load_reference()
    for case in DSTATE_CASES:
        name, seed, batch, dim, L, N, G, tl, has_D, has_z, has_b, sp = case
        d = scan_inputs(seed, batch, dim, L, N, G, tl)
        leaves = {k: d[k].clone().requires_grad_() for k in ("u", "delta", "A", "B", "C", "D", "z", "delta_bias")}
        out, last = ssi.selective_scan_ref(
            leaves["u"], leaves["delta"], leaves["A"], leaves["B"], leaves["C"],
            leaves["D"] if has_D else None, leaves["z"] if has_z else None,
            leaves["delta_bias"] if has_b else None, sp, return_last_state=True)
        res = {"out": out.detach().numpy(), "last_state": last.detach().numpy()}
        keys = ["u", "delta", "A", "B", "C"] + (["D"] if has_D else []) + (["z"] if has_z else []) + (["delta_bias"] if has_b else [])
        grads = torch.autograd.grad(out, [leaves[k] for k in keys], d["dout"])
        for k, g in zip(keys, grads):
            res["d" + k] = g.numpy()
        res["input_checksum"] = np.array([float(d["u"].double().sum()), float(d["B"].double().sum())])
        np.savez_compressed(os.path.join(gg.OUT, f"scan_{name}.npz"), **res)
        print("scan", name, out.shape, float(out.abs().max()))


if __name__ == "__main__":
    main()
