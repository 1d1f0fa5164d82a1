"""Writes tests/golden/fullsize_ref_cuda.npz: what the reference's op sequence on the reference's own CUDA kernels (oracle/_ref,
built by oracle/build_ref.py) computes for the two full-size cases of tests/test_gpu_fullsize.py -- a seeded sample of the
config-2 logits, and loss / global gradient norm of one bf16 training step.  Needs a CUDA device and oracle/_ref.

    python tools/gen_fullsize_golden.py [--out tests/golden/fullsize_ref_cuda.npz]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import test_gpu_fullsize as fs  # noqa: E402
from ref_equivalent_step import bind_reference_kernels  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=fs.GOLDEN)
    args = ap.parse_args()
    from oracle import oracle as orc
    bind_reference_kernels(orc)
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False            # as the test's exact_fp32 fixture
    m = fs.default_model().eval()
    sd = {k: v.detach().clone().contiguous() for k, v in m.state_dict().items()}
    with torch.no_grad():
        logits = fs.sample_logits(orc.segmamba_forward(sd, fs.config2_input()))
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    rp = {k: torch.nn.Parameter(v) for k, v in sd.items()}
    x, y = fs.step_inputs()
    loss, gradnorm = fs.step_loss_and_gradnorm(lambda t: orc.segmamba_forward(rp, t), list(rp.values()), x, y)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, config2_logits=logits.numpy(), step_loss=np.float32(loss), step_gradnorm=np.float32(gradnorm),
             device=torch.cuda.get_device_name(0))
    print("wrote", args.out, "loss", loss, "grad norm", gradnorm)


if __name__ == "__main__":
    main()
