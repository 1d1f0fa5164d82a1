"""Host-side logic of the round-2 wrappers that needs no GPU: operand-major detection and alignment rules of the GEMM wrapper,
its routing table, the split-K heuristic, and the loud failure of the layout / GEMM entry points on CPU tensors (the product has
no CPU path)."""
import pytest
import torch


def test_gemm_operand_major_detection():
    from segmamba_b200 import gemm as G
    a = torch.zeros(64, 48, dtype=torch.bfloat16)
    assert G._operand(a, "A") == (0, 48)                      # K contiguous: K-major, ld = row stride
    assert G._operand(a.t(), "A") == (1, 48)                  # transposed view: first axis contiguous -> MN-major
    wide = torch.zeros(40, 1024, dtype=torch.bfloat16)[:8]    # row slice of a (40, b*l) matrix (x_dbl[:R8])
    assert G._operand(wide, "B") == (0, 1024)
    assert G._operand(wide.t(), "B") == (1, 1024)
    with pytest.raises(RuntimeError):
        G._operand(torch.zeros(16, 12, dtype=torch.bfloat16), "A")          # 24-byte rows: not a TMA pitch
    with pytest.raises(RuntimeError):
        G._operand(torch.zeros(16, 32, dtype=torch.bfloat16)[:, ::2], "A")  # no contiguous axis
    assert not G.supported(a, a)                               # CPU tensors never qualify


def test_gemm_routing_and_split_k():
    from segmamba_b200 import gemm as G
    assert G.MODE in ("auto", "all", "off") and G.SPLIT_TOKENS == 16384
    assert G._split_k_for(524288) == 132 and G._split_k_for(65536) == 128 and G._split_k_for(1000) == 1


def test_gemm_and_layout_raise_on_cpu_tensors():
    from segmamba_b200 import gemm as G
    from segmamba_b200 import layout
    a = torch.zeros(64, 48, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        G.gemm(a, a)
    with pytest.raises(RuntimeError):
        G.linear(torch.zeros(4, 48), torch.zeros(8, 48))       # fp32 without autocast: 16-bit operands only
    x = torch.zeros(1, 8, 4, 4, 4).contiguous(memory_format=torch.channels_last_3d)
    assert not layout.supported(x, x)
    with pytest.raises(RuntimeError):
        layout.cat_channels(x, x)


def test_dense_checkpoint_size_formula():
    """smb_scan_dense_floats: batch x octets x (chunks x 32 blocks) x 8 channels x N states (no GPU needed: host arithmetic)"""
    from segmamba_b200 import _lib
    l = _lib.lib()
    assert l.smb_scan_dense_floats(2, 96, 262144, 16, 1) == 2 * 12 * (1024 * 32) * 8 * 16
    assert l.smb_scan_dense_floats(1, 44, 5003, 16, 1) == 1 * 6 * (20 * 32) * 8 * 16      # partial octet, ragged length
    assert l.smb_scan_dense_floats(2, 48, 2048, 8, 2) == 2 * (3 * 2) * (8 * 32) * 8 * 8    # two B/C groups of 24 channels
    assert l.smb_scan_dense_floats(2, 45, 100, 16, 2) == 0                                 # dim not divisible by the groups
