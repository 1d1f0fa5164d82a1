"""segmamba_b200 -- H100-native (sm_90a) implementation of the SegMamba hot path.

Public surface (mirrors the reference's, see INTEGRATION.md):

    segmamba_b200.selective_scan_cuda      drop-in for the pybind module `selective_scan_cuda`
    segmamba_b200.causal_conv1d_cuda       drop-in for the pybind module `causal_conv1d_cuda`
    segmamba_b200.selective_scan_interface selective_scan_fn, causal_conv1d_fn, mamba_inner_fn_no_out_proj
    segmamba_b200.mamba_simple.Mamba       the tri-directional (bimamba_type="v3") mixer
    segmamba_b200.segmamba.SegMamba        the model (same constructor, forward and state_dict)

`install_dropin()` registers the two operator modules under the reference's import names so that the
reference's own Python (mamba_ssm/ops/selective_scan_interface.py, mamba_simple.py, segmamba.py, 3_train.py,
4_predict.py) runs unchanged on the native kernels.
"""
import sys

__version__ = "0.1.0"


def install_dropin(force: bool = False) -> None:
    """Make `import selective_scan_cuda` / `import causal_conv1d_cuda` resolve to the native shims."""
    from . import causal_conv1d_cuda, selective_scan_cuda
    for name, mod in (("selective_scan_cuda", selective_scan_cuda), ("causal_conv1d_cuda", causal_conv1d_cuda)):
        if force or name not in sys.modules:
            sys.modules[name] = mod
