"""BASELINE-size parity cases (seconds each on an H100):
  * config 2 (SURVEY.md section 8d): the default SegMamba on one 4x128^3 patch, fp32, eval -- native module vs the reference's
    op sequence (oracle.segmamba_forward: NCDHW, flips / stack / rearrange copies, ATen norms) running on the reference's OWN CUDA
    kernels (oracle/_ref, built by oracle/build_ref.py), same state_dict.  What the reference kernels computed is stored in
    tests/golden/fullsize_ref_cuda.npz (a seeded sample of the logits; written by tools/gen_fullsize_golden.py on an H100);
  * fused instance norm at the largest activation of the model (2, 48, 128^3) against fp32 torch;
  * one bf16 training step at full size: loss and global gradient norm of the native module against the stored ones of the
    reference-kernel step, and the two native backward paths against each other."""
import os

import numpy as np
import pytest
import torch

from util import assert_close

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fullsize_ref_cuda.npz")
N_SAMPLE = 1 << 16


def default_model():
    from segmamba_b200.segmamba import SegMamba
    torch.manual_seed(0)
    return SegMamba(in_chans=4, out_chans=4, depths=[2, 2, 2, 2], feat_size=[48, 96, 192, 384]).cuda()


def config2_input():
    return torch.rand(1, 4, 128, 128, 128, generator=torch.Generator().manual_seed(11)).cuda()             # 0_inference.py:6


def sample_logits(t):
    idx = torch.randint(0, t.numel(), (N_SAMPLE,), generator=torch.Generator().manual_seed(12))
    return t.detach().reshape(-1)[idx.to(t.device)].float().cpu()


def step_inputs():
    g = torch.Generator().manual_seed(13)
    return torch.rand(2, 4, 128, 128, 128, generator=g).cuda(), torch.randint(0, 4, (2, 128, 128, 128), generator=g).cuda()


@pytest.fixture
def exact_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_config2_default_model_128_fp32_vs_reference_cuda(exact_fp32):
    m = default_model().eval()
    with torch.no_grad():
        out = m(config2_input())
    assert out.shape == (1, 4, 128, 128, 128)
    ref = torch.from_numpy(np.load(GOLDEN)["config2_logits"])
    assert_close(sample_logits(out), ref, 1e-3, "config 2 logits vs the reference op sequence on the reference CUDA kernels")


@pytest.mark.parametrize("mode", ["plain", "residual", "two_norms"])
def test_fused_instance_norm_largest_activation(mode):
    from segmamba_b200.instance_norm import fused_instance_norm
    import torch.nn.functional as F
    torch.manual_seed(1)
    shape = (2, 48, 128, 128, 128)
    x = (torch.randn(shape, device="cuda") * 2 + 0.5).bfloat16().contiguous(memory_format=torch.channels_last_3d).requires_grad_()
    x2 = torch.randn(shape, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last_3d).requires_grad_()
    dy = torch.randn(shape, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last_3d)
    if mode == "plain":
        y = fused_instance_norm(x, "leaky_relu", 0.01)
        ins = [x]
    elif mode == "residual":
        y = fused_instance_norm(x, "leaky_relu", 0.01, add=x2)
        ins = [x, x2]
    else:
        y = fused_instance_norm(x, "leaky_relu", 0.01, add=x2, add_norm=True)
        ins = [x, x2]
    g = torch.autograd.grad(y, ins, dy, retain_graph=True)
    xr, x2r = x.detach().float().requires_grad_(), x2.detach().float().requires_grad_()
    t = F.instance_norm(xr, eps=1e-5)
    if mode == "residual":
        t = t + x2r
    elif mode == "two_norms":
        t = t + F.instance_norm(x2r, eps=1e-5)
    yr = F.leaky_relu(t, 0.01)
    gr = torch.autograd.grad(yr, [xr, x2r][:len(ins)], dy.float(), retain_graph=True)
    assert_close(y, yr, 1e-2, "y")
    # LeakyReLU kink: with two operands t = IN(x) + ... cancels to |t| ~ 1e-7 at a handful of the 2e8 voxels, where two
    # fp32-accurate evaluations may disagree on the sign of t and the incoming gradient is scaled by 1 or by 0.01.  Those
    # voxels are compared through the channel statistics only (their dy is zeroed on both sides); a single-operand t = IN(x)
    # of bf16 data never comes that close to zero.
    if mode != "plain":
        keep = (t.detach().abs() > 1e-3).to(dy.dtype)
        dyk = dy * keep
        g = torch.autograd.grad(y, ins, dyk)
        gr = torch.autograd.grad(yr, [xr, x2r][:len(ins)], dyk.float())
    for a, b, n in zip(g, gr, ("dx", "dx2")):
        assert_close(a, b, 2e-2, n)


def step_loss_and_gradnorm(forward, params, x, y):
    for p in params:
        p.grad = None
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = torch.nn.functional.cross_entropy(forward(x).float(), y)
    loss.backward()
    gn = torch.nn.utils.clip_grad_norm_(params, 1e9)
    return float(loss), float(gn)


def test_full_size_bf16_training_step_vs_reference_kernels():
    from segmamba_b200 import selective_scan_cuda as ssc
    m = default_model().train()
    x, y = step_inputs()
    params = list(m.parameters())
    la, ga = step_loss_and_gradnorm(m, params, x, y)
    old = ssc.LOW_MEMORY_BWD
    try:
        ssc.LOW_MEMORY_BWD = not old
        lb, gb = step_loss_and_gradnorm(m, params, x, y)
    finally:
        ssc.LOW_MEMORY_BWD = old
    gold = np.load(GOLDEN)
    lr, gr = float(gold["step_loss"]), float(gold["step_gradnorm"])
    print(f"full-size bf16 step: loss native {la:.5f} / other backward path {lb:.5f} / reference kernels {lr:.5f}; "
          f"grad norm {ga:.4f} / {gb:.4f} / {gr:.4f}")
    assert abs(la - lb) <= 1e-3 * abs(la) and abs(ga - gb) <= 1e-2 * ga
    assert abs(la - lr) <= 1e-2 * abs(lr), (la, lr)
    assert abs(ga - gr) <= 3e-2 * gr, (ga, gr)
