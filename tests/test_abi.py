"""CPU-side checks of the C-ABI boundary: the shared library loads and exports exactly the symbols the header declares,
the ctypes structures match the header's field lists, and the product fails loudly without a GPU / library."""
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "segmamba_b200.h")


def _header_functions():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"SMB_API\s+[\w\s\*]+?\b(smb_\w+)\s*\(", src)))


def _header_struct_fields(name):
    src = open(HEADER).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for stmt in body.split(";"):
        stmt = stmt.strip()
        if not stmt:
            continue
        decl = re.sub(r"^(const\s+)?(void|float|int32_t|int64_t|size_t)\s*", "", stmt)
        for part in decl.split(","):
            fields.append(part.replace("*", "").strip())
    return fields


def test_library_exports_match_header():
    import __graft_entry__ as ge
    from segmamba_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        ge.build()
    funcs = _header_functions()
    assert funcs, "no SMB_API declarations found"
    assert sorted(_lib.EXPORTS.keys()) == funcs
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = sorted(set(re.findall(r"\sT\s+(smb_\w+)", out)))
    assert exported == funcs
    l = _lib.lib()                       # loads and binds every symbol (no compute calls)
    assert l.smb_version() >= 100
    assert l.smb_scan_fwd_workspace_bytes(1, 96, 262144, 16) > 0


@pytest.mark.parametrize("cname,pyname", [("smb_scan_fwd_args", "ScanFwdArgs"), ("smb_scan_bwd_args", "ScanBwdArgs"),
                                          ("smb_conv1d_args", "Conv1dArgs"), ("smb_conv1d_bwd_args", "Conv1dBwdArgs"),
                                          ("smb_seq_permute_args", "SeqPermuteArgs"), ("smb_instnorm_args", "InstNormArgs"),
                                          ("smb_instnorm_bwd_args", "InstNormBwdArgs"), ("smb_layernorm_args", "LayerNormArgs"),
                                          ("smb_layernorm_bwd_args", "LayerNormBwdArgs")])
def test_ctypes_structs_match_header(cname, pyname):
    from segmamba_b200 import _lib
    py = [f[0] for f in getattr(_lib, pyname)._fields_]
    assert py == _header_struct_fields(cname)


def test_sm90a_sass_present():
    """the library carries sm_90a SASS (cuobjdump lists the arch) -- built for H100, not a generic PTX blob."""
    from segmamba_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback():
    """CPU tensors must raise, never silently compute (SURVEY.md: the hot path has no CPU implementation)."""
    from segmamba_b200 import causal_conv1d_cuda, selective_scan_cuda
    u = torch.randn(1, 4, 32)
    A = -torch.rand(4, 16)
    B = torch.randn(1, 1, 16, 32)
    with pytest.raises(RuntimeError):
        selective_scan_cuda.fwd(u, u, A, B, B, None, None, None, False)
    with pytest.raises(RuntimeError):
        causal_conv1d_cuda.causal_conv1d_fwd(u, torch.randn(4, 4), None, True)
    with pytest.raises(RuntimeError):
        causal_conv1d_cuda.causal_conv1d_update(u[:, :, 0], torch.zeros(1, 4, 4), torch.randn(4, 4), None, True)
    from segmamba_b200.instance_norm import fused_instance_norm
    from segmamba_b200.layer_norm import fused_layer_norm
    with pytest.raises(RuntimeError):
        fused_instance_norm(torch.randn(1, 8, 4, 4, 4))
    with pytest.raises(RuntimeError):
        fused_layer_norm(torch.randn(16, 48), torch.ones(48), torch.zeros(48))


def test_missing_library_fails_loudly(monkeypatch):
    from segmamba_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libsegmamba_b200.so")
    with pytest.raises(RuntimeError, match="no fallback"):
        _lib.lib()


def test_product_does_not_import_oracle():
    """only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
    pkg = os.path.join(ROOT, "segmamba_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("checker", ""), f"{f} mentions the oracle"


def test_install_dropin():
    import sys
    import segmamba_b200
    saved = {k: sys.modules.pop(k, None) for k in ("selective_scan_cuda", "causal_conv1d_cuda")}
    try:
        segmamba_b200.install_dropin()
        import causal_conv1d_cuda
        import selective_scan_cuda
        assert callable(selective_scan_cuda.fwd) and callable(selective_scan_cuda.bwd)
        assert callable(causal_conv1d_cuda.causal_conv1d_fwd) and callable(causal_conv1d_cuda.causal_conv1d_bwd)
    finally:
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
