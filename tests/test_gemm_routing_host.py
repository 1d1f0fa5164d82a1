"""Routing of every pointwise product of the default model (bench.py: batch 2, 4x128^3 patches, feat_size 48 / 96 / 192 / 384)
through ``gemm.plan`` in the three SMB_GEMM modes, on ``meta`` operands laid out as the model's code passes them."""
import math

import pytest
import torch

BF = torch.bfloat16
STAGES = [(48, 2 * 64 ** 3), (96, 2 * 32 ** 3), (192, 2 * 16 ** 3), (384, 2 * 8 ** 3)]      # (C, mixer tokens)
# 1x1x1 convolutions outside the stages: UnetResBlock.conv3 of encoder1..5 and of decoder5..2 (C_in, C_out, tokens)
RES_CONV3 = [(4, 48, 2 * 128 ** 3), (48, 96, 2 * 64 ** 3), (96, 192, 2 * 32 ** 3), (192, 384, 2 * 16 ** 3),
             (384, 768, 2 * 8 ** 3), (768, 384, 2 * 16 ** 3), (384, 192, 2 * 32 ** 3), (192, 96, 2 * 64 ** 3),
             (96, 48, 2 * 128 ** 3)]


def k_major(rows, cols, dtype=BF, device="meta"):
    return torch.empty_strided((rows, cols), (cols, 1), dtype=dtype, device=device)


def mn_major(rows, cols, dtype=BF):
    return k_major(cols, rows, dtype).t()


def mixer_products(C, T):
    """(name, x, y, tokens) of every product of one Mamba layer, as Mamba.forward / MambaInnerFnNoOutProj / _MatmulNT pass them."""
    di, R8 = 2 * C, math.ceil(math.ceil(C / 16) / 8) * 8
    NX = R8 + 32
    return [
        ("in_proj", k_major(4 * C, C), k_major(T, C), 0),
        ("in_proj.dW", k_major(4 * C, T), mn_major(C, T), T),
        ("in_proj.dX", mn_major(T, 4 * C), mn_major(C, 4 * C), 4 * C),
        ("out_proj", mn_major(T, di), k_major(C, di), 0),
        ("out_proj.dX", mn_major(di, C), k_major(T, C), C),
        ("out_proj.dW", mn_major(C, T), k_major(di, T), T),
        ("x_proj", k_major(NX, di), mn_major(T, di), 0),
        ("dt_proj", k_major(di, R8), mn_major(T, R8), 0),
        ("dt_proj.dW", k_major(di, T), k_major(R8, T), T),
        ("dx_dbl[:R8]", k_major(R8, di), mn_major(T, di), 0),
        ("x_proj.dW", k_major(NX, T), k_major(di, T), T),
        ("dconv2", mn_major(di, NX), mn_major(T, NX), 0),
    ]


def conv1x1s():
    """(name, C_in, C_out, tokens) of every 1x1x1 convolution: GSC.proj3 / proj4 and MlpChannel.fc1 / fc2 per stage, and the
    residual convolutions"""
    out = []
    for i, (C, T) in enumerate(STAGES):
        out += [(f"gsc{i}.proj3", C, C, T), (f"gsc{i}.proj4", C, C, T), (f"mlp{i}.fc1", C, 2 * C, T), (f"mlp{i}.fc2", 2 * C, C, T)]
    return out + [(f"res{j}.conv3", ci, co, T) for j, (ci, co, T) in enumerate(RES_CONV3)]


def conv_products(ci, co, T):
    """conv1x1's forward decision (fp32 weight, bf16 compute), then _Linear's products once it is native"""
    return [("fwd", k_major(T, ci), k_major(co, ci, torch.float32), 0, BF),
            ("dX", k_major(T, co), mn_major(ci, co), 0, None),
            ("dW", mn_major(co, T), mn_major(ci, T), T, None)]


@pytest.fixture
def G(monkeypatch):
    from segmamba_b200 import gemm
    return lambda mode: (monkeypatch.setattr(gemm, "MODE", mode), gemm)[1]


def test_auto_routes_the_token_contractions_of_stages_0_and_1(G):
    g = G("auto")
    for i, (C, T) in enumerate(STAGES):
        for name, x, y, tokens in mixer_products(C, T):
            want = ({48: 132, 96: 128}[C], torch.float32) if name.endswith(".dW") and i < 2 else None
            assert g.plan(x, y, tokens) == want, (i, name)
    for name, ci, co, T in conv1x1s():
        x, w = conv_products(ci, co, T)[0][1:3]
        assert g.plan(x, w, 0, BF) is None, name            # so the whole convolution stays on cuDNN


def test_all_routes_every_product_the_kernel_takes(G):
    g = G("all")
    for C, T in STAGES:
        for name, x, y, tokens in mixer_products(C, T):
            assert g.plan(x, y, tokens) == ((g._split_k_for(T), torch.float32) if tokens >= 16384 else (1, None)), (C, name)
    for name, ci, co, T in conv1x1s():
        for what, x, y, tokens, dtype in conv_products(ci, co, T):
            want = None if ci % 8 else (g._split_k_for(T), torch.float32) if tokens >= 16384 else (1, None)
            assert g.plan(x, y, tokens, dtype) == want, (name, what)
            if want is None:
                break                                        # C_in = 4: the input convolution stays on cuDNN


def test_off_routes_nothing(G):
    g = G("off")
    for C, T in STAGES:
        for name, x, y, tokens in mixer_products(C, T):
            assert g.plan(x, y, tokens) is None, (C, name)
    for name, ci, co, T in conv1x1s():
        for what, x, y, tokens, dtype in conv_products(ci, co, T):
            assert g.plan(x, y, tokens, dtype) is None, (name, what)


@pytest.mark.parametrize("mode", ["auto", "all"])
def test_products_the_kernel_cannot_take_go_to_the_library(G, mode):
    g = G(mode)
    T = 2 * 64 ** 3
    assert g.plan(k_major(192, T), mn_major(48, T), T) is not None
    assert g.plan(k_major(192, T, torch.float32), mn_major(48, T, torch.float32), T) is None       # fp32 / no autocast
    assert g.plan(k_major(192, T), mn_major(48, T, torch.float32), T) is None                      # mixed dtypes
    assert g.plan(k_major(T, 48, torch.float32), k_major(96, 48, torch.float32), 0, torch.float32) is None
    assert g.plan(k_major(192, T), mn_major(44, T), T) is None                                    # 88-byte rows (44 % 8)
    assert g.plan(k_major(T, 12), k_major(96, 12), 0, BF) is None                                 # 24-byte rows
    cpu = [k_major(192, 16384, device="cpu"), k_major(48, 16384, device="cpu")]
    assert g.plan(*cpu, 16384) is not None and g.route(*cpu, 16384) is None                       # CPU tensors
    big = [k_major(2048, T), k_major(2048, T)]                                                     # 2^22 outputs: no split-K
    assert g.plan(*big, T) == ((1, None) if mode == "all" else None)
