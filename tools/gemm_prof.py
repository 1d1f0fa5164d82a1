"""Where a smb_gemm launch waits: cycles per role inside barrier waits (SMB_GEMM_PROF counters), for a few shapes."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from segmamba_b200 import gemm as G
bf = torch.bfloat16
r = lambda *s: torch.randn(*s, device="cuda").to(bf)
T = 524288
cases = [("in_proj W[192,48] x X[T,48]", r(192, 48), r(T, 48)),
         ("X[T,48] x W[192,48] (tokens as M)", r(T, 48), r(192, 48)),
         ("x_proj Wx[40,96] x U^T (MN)", r(40, 96), r(96, T).t()),
         ("dt dx: Wdt^T[8,96](MN) x dd^T (MN)", r(96, 8).t(), r(96, T).t()),
         ("out_proj Y^T (MN) x Wo[48,96]", r(96, T).t(), r(48, 96))]
prof = torch.zeros(16, dtype=torch.int64, device="cuda")
for name, a, b in cases:
    for _ in range(2):
        G.gemm(a, b)
    torch.cuda.synchronize()
    prof.zero_()
    os.environ["SMB_GEMM_PROF"] = str(prof.data_ptr())
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); G.gemm(a, b); e.record(); torch.cuda.synchronize()
    del os.environ["SMB_GEMM_PROF"]
    c = prof.tolist()
    M, K = a.shape; N = b.shape[0]
    tiles = ((M + 127) // 128) * ((N + 255) // 256 if N > 256 else 1)
    ctas = min(tiles, torch.cuda.get_device_properties(0).multi_processor_count) * 1e3
    print(f"{name}: {s.elapsed_time(e)*1e3:.1f} us; per-CTA kcycles ({ctas / 1e3:.0f} CTAs): first consumer warp total {c[7]/ctas:.1f}  "
          f"producer-wait-empty {c[0]/ctas:.1f}  consumer-wait-full {c[2]/ctas:.1f}  epilogue {c[11]/ctas:.1f}  tiles {tiles}")
