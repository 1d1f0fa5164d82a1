"""The tri-directional mixer (Mamba, MambaLayer) in 16 bits at the training step's stage shapes, against fp64.

The training step runs the mixer under bf16 autocast at batch 2.  There, and only there, it takes paths that the fp32 goldens at
1024 tokens never reach: split-K weight gradients on the native GEMM (from SPLIT_TOKENS tokens on) whose operands are the mixer's
own strided views, 16-bit scans whose B / C are row slices of one (R8 + 2N, b*L) matrix (batch stride L below state stride b*L:
the swapped TMA map), channel-major u / delta / z, and the zero-padded dt rank (3 -> 8, 6 -> 8, 12 -> 16).

Inputs: the module's own initialisation; every parameter, the input and dout rounded to bf16 values with |v| < 2^-14 flushed to
zero, so that they are exact in fp16 too and autocast's casts are exact.  One fp64 reference then serves both dtypes and both
GEMM modes.

* Layer 1 records every native call of one forward and backward (gemm, scan fwd_ex / bwd_ex, conv1d fwd / bwd, seq_permute) with
  clones of its operands taken before the call, and replays each against fp64 on those operands: ``x @ y.T`` in fp64, the fp64
  C oracle (in walk order), the torch indexing of the slice permutation.  It also asserts that the claimed paths ran.
* Layer 2 compares the module's output, input gradient and every parameter gradient with ``oracle.mamba_v3_forward`` on float64
  copies, in max-norm relative error (the project's TOL / GRAD_TOL) and normwise relative error ||a - b||_F / ||b||_F, which is
  where an error confined to one parameter stands out from rounding noise.
* Layer 3 shows both layers are sharp: a split-K product with its last K slice dropped, and a 1 % error in one gradient.

Normwise error, worst case over CASES, measured on one NVIDIA H100 80GB HBM3 (power limit 700 W); NORM_TOL is about 3x these:

    tensor class      bf16     fp16        tensor class      bf16     fp16
    out               4.4e-3   5.4e-4      dt_proj.weight    7.5e-3   8.4e-4
    dx                4.5e-3   5.6e-4      dt_proj.bias      6.4e-3   7.5e-4
    in_proj.weight    4.7e-3   5.5e-4      A_log             5.9e-3   5.6e-4
    conv1d.weight     4.8e-3   5.1e-4      D                 4.3e-3   4.6e-4
    conv1d.bias       3.9e-3   4.6e-4      out_proj.weight   4.5e-3   5.4e-4
    x_proj.weight     8.4e-3   7.7e-4      norm.weight/bias  4.9e-3 / 4.0e-3 (bf16 only)

Every fp16 error is 8-10x below its bf16 one, the ratio of the two significands (2^-11 vs 2^-8): the floor is the rounding of
the 16-bit activations, not a systematic error.  In bf16 it sits at about half a percent, so there the normwise check finds an
error of a few percent in one tensor but not one of 1 % (the scaled gradient below measured 1.2e-2 against 6.4e-3 for its
twins); the 1 % sharpness test therefore runs in fp16.  The whole file takes 7 to 9 minutes, almost all of it the fp64 C
oracle on 8 CPU cores.
"""
import copy
import inspect
import re

import pytest
import torch
import torch.nn.functional as F

from util import GRAD_TOL, TOL, rel_err

pytestmark = pytest.mark.gpu

# (d_model, L, nslices) of the four encoder stages of the default model (feat_size 48 / 96 / 192 / 384 on a 128^3 patch)
STAGES = {0: (48, 262144, 64), 1: (96, 32768, 32), 2: (192, 4096, 16), 3: (384, 512, 8)}
BF16, F16 = torch.bfloat16, torch.float16


class Case:
    def __init__(self, name, d_model, L, nslices, batch=2, d_state=16, dtype=BF16, mode="auto", layer=False, streams=False,
                 stash=False):
        self.name, self.d_model, self.L, self.nslices, self.batch, self.d_state = name, d_model, L, nslices, batch, d_state
        self.dtype, self.mode, self.layer, self.streams, self.stash = dtype, mode, layer, streams, stash
        # cases with the same key share the module, the inputs and the fp64 reference
        self.key = (d_model, L, nslices, batch, d_state, layer)

    @property
    def tokens(self):
        return self.batch * self.L


def _stage(s, **kw):
    d_model, L, ns = STAGES[s]
    tag = "".join(f"-{k}" for k in ("streams", "stash") if kw.get(k)) + (f"-n{kw['d_state']}" if "d_state" in kw else "")
    dt = {BF16: "bf16", F16: "f16"}[kw.get("dtype", BF16)]
    return Case(f"{'layer' if kw.get('layer') else 'mamba'}-s{s}{tag}-{dt}-{kw.get('mode', 'auto')}", d_model, L, ns, **kw)


# ordered so that cases sharing a reference are adjacent (one reference is kept alive at a time)
CASES = ([_stage(0)]
         + [_stage(1, mode=md) for md in ("auto", "all")] + [_stage(1, dtype=F16)]
         + [_stage(1, streams=True), _stage(1, stash=True)]
         + [_stage(1, d_state=32), _stage(1, d_state=64)]
         + [_stage(2, mode=md) for md in ("auto", "all")]
         + [_stage(3, dtype=dt, mode=md) for dt in (BF16, F16) for md in ("auto", "all")]
         # b*L = 24585 is not a multiple of 8: no GEMM operand has 16-byte rows and the scans' B / C take the untiled path
         + [Case("mamba-ragged-b3-bf16-auto", 40, 8195, 5, batch=3)]
         # the stage-0 layer would add a second stage-0 reference (minutes of fp64 CPU time) for the LayerNorm and residual only
         + [_stage(1, layer=True)])

# normwise relative error bounds per tensor class, about 3x the worst case measured over CASES (module docstring).  Every bf16
# bound is above 5e-3: each bf16 activation, scan output and GEMM output carries a 2^-9 relative rounding, and the measured
# bf16 errors are 8-10x the fp16 ones, as that rounding predicts.
NORM_TOL = {
    BF16: {"out": 1.5e-2, "dx": 1.5e-2, "in_proj.weight": 1.5e-2, "conv1d.weight": 1.5e-2, "conv1d.bias": 1.2e-2,
           "x_proj.weight": 2.5e-2, "dt_proj.weight": 2.5e-2, "dt_proj.bias": 2e-2, "A_log": 2e-2, "D": 1.5e-2,
           "out_proj.weight": 1.5e-2, "norm.weight": 1.5e-2, "norm.bias": 1.2e-2},
    F16: {"out": 1.6e-3, "dx": 1.7e-3, "in_proj.weight": 1.7e-3, "conv1d.weight": 1.5e-3, "conv1d.bias": 1.4e-3,
          "x_proj.weight": 2.3e-3, "dt_proj.weight": 2.5e-3, "dt_proj.bias": 2.3e-3, "A_log": 1.7e-3, "D": 1.4e-3,
          "out_proj.weight": 1.6e-3},
}


# --------------------------------------------------------------------------------------------------------------------- inputs
def _q(t):
    """bf16 value, zero below 2^-14: exact in bf16 and in fp16"""
    t = t.detach().bfloat16().float()
    return torch.where(t.abs() < 2.0 ** -14, torch.zeros_like(t), t)


def _inputs(c):
    """CPU module (fp32 storage of bf16 values) with its own initialisation, input and dout"""
    from segmamba_b200.mamba_simple import Mamba
    from segmamba_b200.segmamba import MambaLayer
    seed = c.d_model * 7 + c.d_state + c.batch
    torch.manual_seed(seed)
    if c.layer:
        m = MambaLayer(dim=c.d_model, d_state=c.d_state, num_slices=c.nslices)
        s = round(c.L ** (1 / 3))
        assert s ** 3 == c.L
        shape = (c.batch, c.d_model, s, s, s)
    else:
        m = Mamba(d_model=c.d_model, d_state=c.d_state, nslices=c.nslices)
        shape = (c.batch, c.L, c.d_model)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(_q(p))
    g = torch.Generator().manual_seed(seed + 1)
    return m, _q(torch.randn(shape, generator=g)), _q(torch.randn(shape, generator=g))


def _reference(c, m, x, dout):
    """oracle.mamba_v3_forward (+ LayerNorm and residual for MambaLayer) on float64 copies: (out, {name: grad}) on the CPU"""
    from oracle import oracle as orc
    p = {k: v.detach().double().requires_grad_() for k, v in m.state_dict().items()}
    xo = x.double().requires_grad_()
    if c.layer:
        B, C = x.shape[:2]
        xn = F.layer_norm(xo.reshape(B, C, -1).transpose(-1, -2), (C,), p["norm.weight"], p["norm.bias"], m.norm.eps)
        ro = orc.mamba_v3_forward(p, xn, c.nslices, prefix="mamba.").transpose(-1, -2).reshape(x.shape) + xo
    else:
        ro = orc.mamba_v3_forward(p, xo, c.nslices)
    names = [n for n, _ in m.named_parameters()]
    grads = torch.autograd.grad(ro, [xo] + [p[n] for n in names], dout.double())
    return ro.detach(), dict(zip(["x"] + names, grads))


_ref_cache = {}


def _case_data(c):
    if c.key not in _ref_cache:
        _ref_cache.clear()                          # the stage-0 reference is a few GB of host memory: one alive at a time
        m, x, dout = _inputs(c)
        _ref_cache[c.key] = (m, x, dout, _reference(c, m, x, dout))
    return _ref_cache[c.key]


# ---------------------------------------------------------------------------------------------------------------- recording
class Call:
    def __init__(self, op, args, layout, result):
        self.op, self.args, self.layout, self.result = op, args, layout, result


def _clone(v):
    if isinstance(v, torch.Tensor):
        return v.detach().clone()                   # clone() keeps the strides of a dense view
    if isinstance(v, (tuple, list)):
        return type(v)(_clone(e) for e in v)
    return v


class Recorder:
    """wraps the native entry points on the module attributes their callers look up at call time"""

    ENTRIES = (("gemm", "gemm"), ("selective_scan_cuda", "fwd_ex"), ("selective_scan_cuda", "bwd_ex"),
               ("causal_conv1d_cuda", "causal_conv1d_fwd_ex"), ("causal_conv1d_cuda", "causal_conv1d_bwd_ex"),
               ("causal_conv1d_cuda", "seq_permute"))

    def __init__(self, monkeypatch):
        import importlib
        self.calls = []
        for mod_name, fn_name in self.ENTRIES:
            mod = importlib.import_module("segmamba_b200." + mod_name)
            monkeypatch.setattr(mod, fn_name, self._wrap(fn_name, getattr(mod, fn_name)))

    def _wrap(self, op, fn):
        sig = inspect.signature(fn)

        def call(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            layout = {k: (tuple(v.shape), v.stride()) for k, v in bound.arguments.items() if isinstance(v, torch.Tensor)}
            # inputs are cloned before the call: out= and accumulate= write in place
            saved = {k: (None if k in ("hstates", "hdense") else _clone(v)) for k, v in bound.arguments.items()}
            res = fn(*args, **kwargs)
            # outputs are cloned at once: later calls write into some of them (dconv2 is a view of the scan's du)
            self.calls.append(Call(op, saved, layout, _clone(res)))
            return res
        return call

    def of(self, op):
        return [c for c in self.calls if c.op == op]


# ------------------------------------------------------------------------------------------------------- layer 1: replay
def _walk(direction):
    return (lambda t: t.flip(-1)) if direction else (lambda t: t)


def _host(t):
    return None if t is None else t.detach().cpu().float()


def check_gemm(a, res):
    """fp64 x @ y.T (+ the prior out when accumulating); fp32 outputs (split-K) to 1e-4, 16-bit ones to one output rounding"""
    from segmamba_b200.gemm import EPI_NONE
    assert a["epilogue"] == EPI_NONE and a["bias"] is None, "the mixer's products have no epilogue"
    ref = a["a"].double() @ a["b"].double().t()
    if a["accumulate"]:
        ref += a["out"].double()
    return [("gemm", rel_err(res, ref), 1e-4 if res.dtype == torch.float32 else 8e-3)]


def check_scan_fwd(a, res):
    from oracle import oracle as orc
    f = _walk(a["direction"])
    h = {k: _host(a[k]) for k in ("u", "delta", "A", "B", "C", "D_", "z_", "delta_bias_")}
    y, oz, _, _ = orc.selective_scan_fwd_raw(f(h["u"]), f(h["delta"]), h["A"], f(h["B"]), f(h["C"]), h["D_"],
                                             None if h["z_"] is None else f(h["z_"]), h["delta_bias_"], a["delta_softplus"])
    tol = TOL[a["u"].dtype]
    out = [("out_z", rel_err(res[2], f(oz)), tol)] if res[2] is not None else []
    if res[0] is not None:
        out.append(("out", rel_err(res[0], f(y)), tol))
    return out


def check_scan_bwd(a, res):
    from oracle import oracle as orc
    f = _walk(a["direction"])
    h = {k: _host(a[k]) for k in ("u", "delta", "A", "B", "C", "D_", "z_", "delta_bias_", "dout")}
    g = orc.selective_scan_bwd_raw(f(h["u"]), f(h["delta"]), h["A"], f(h["B"]), f(h["C"]), h["D_"], f(h["z_"]),
                                   h["delta_bias_"], a["delta_softplus"], f(h["dout"]))
    tol = GRAD_TOL[a["u"].dtype]
    names = ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias", "dz")
    walked = ("du", "ddelta", "dB", "dC", "dz")
    return [(k, rel_err(r, f(g[k]) if k in walked else g[k]), tol) for k, r in zip(names, res) if r is not None]


def check_conv_fwd(a, res):
    from oracle import oracle as orc
    f = _walk(a["direction"])
    o = orc.causal_conv1d_fwd_raw(f(_host(a["x"])), _host(a["weight"]), _host(a["bias_"]), a["silu_activation"])
    return [("out", rel_err(res, f(o)), TOL[a["x"].dtype])]


def check_conv_bwd(a, res):
    from oracle import oracle as orc
    f = _walk(a["direction"])
    dx, dw, db = orc.causal_conv1d_bwd_raw(f(_host(a["x"])), _host(a["weight"]), _host(a["bias_"]), f(_host(a["dout"])),
                                           a["silu_activation"])
    tol = GRAD_TOL[a["x"].dtype]
    out = [("dx", rel_err(res[0], f(dx)), tol), ("dweight", rel_err(res[1], dw), tol)]
    if res[2] is not None:
        out.append(("dbias", rel_err(res[2], db), tol))
    return out


def check_seq_permute(a, res):
    """the reference's indexing (mamba_simple.py:245-247 forward, :261 inverse), bitwise"""
    x, ns = a["src"], a["nslices"]
    assert a["out"] is None and not a["accumulate"], "the mixer permutes into fresh tensors"
    L = x.shape[-1]
    if a["inverse"]:
        ref = x.reshape(*x.shape[:-1], L // ns, ns).transpose(-1, -2).flatten(-2)
    else:
        ref = torch.stack(x.chunk(ns, dim=-1), dim=-1).flatten(-2)
    return [("permute (mismatching elements)", float((res != ref).sum()), 0.0)]


CHECKS = {"gemm": check_gemm, "fwd_ex": check_scan_fwd, "bwd_ex": check_scan_bwd, "causal_conv1d_fwd_ex": check_conv_fwd,
          "causal_conv1d_bwd_ex": check_conv_bwd, "seq_permute": check_seq_permute}


def replay(calls):
    """[(i, op, what, err, tol)] for every output of every recorded call"""
    rows = []
    for i, c in enumerate(calls):
        for what, err, tol in CHECKS[c.op](c.args, c.result):
            rows.append((i, c.op, what, err, tol))
    return rows


def check_coverage(c, rec):
    """the paths the case claims to cover did run"""
    from segmamba_b200 import gemm as G
    gemms = rec.of("gemm")
    if c.tokens % 8:
        assert not gemms, f"{len(gemms)} native GEMM calls with b*L = {c.tokens} (rows not 16-byte aligned)"
    elif c.tokens >= G.SPLIT_TOKENS:
        # dW of in_proj and out_proj, and of x_proj and dt_proj in each of the three directions
        split = [g for g in gemms if g.args["split_k"] > 1]
        assert len(split) >= 8, f"only {len(split)} split-K GEMM calls"
        assert all(g.result.dtype == torch.float32 for g in split)
    if c.mode == "all" and c.tokens % 8 == 0:
        assert any(g.args["split_k"] == 1 for g in gemms), "no single-pass GEMM call in 'all' mode"
    fwd, bwd = rec.of("fwd_ex"), rec.of("bwd_ex")
    assert len(fwd) == 3 and len(bwd) == 3, (len(fwd), len(bwd))
    assert sorted(s.args["direction"] for s in fwd) == [0, 0, 1]
    for s in fwd + bwd:
        assert s.args["u"].dtype == c.dtype
        (_, u_st), (_, b_st), (_, c_st) = s.layout["u"], s.layout["B"], s.layout["C"]
        assert u_st[0] == c.L and u_st[1] == c.tokens, f"u is not channel-major: strides {u_st}"
        if c.batch >= 2:
            assert b_st[0] < b_st[2] and c_st[0] < c_st[2], f"B / C strides {b_st} / {c_st}: not row slices of one matrix"
    assert len(rec.of("causal_conv1d_fwd_ex")) == 3 and len(rec.of("causal_conv1d_bwd_ex")) == 3
    assert len(rec.of("seq_permute")) >= 4


# -------------------------------------------------------------------------------------------------- layer 2: end to end
def tensor_class(name):
    """'mamba.x_proj_s.weight' -> 'x_proj.weight', 'A_b_log' -> 'A_log': the three directions share one bound"""
    return re.sub(r"_(b|s)(?=[._]|$)", "", name[len("mamba."):] if name.startswith("mamba.") else name)


def norm_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, f"shape {tuple(a.shape)} vs {tuple(b.shape)}"
    nb = float(torch.linalg.vector_norm(b))
    return float(torch.linalg.vector_norm(a - b)) / (nb if nb > 0 else 1.0)


def end_to_end(out, grads, ref, dtype):
    """[(tensor, class, max-norm err, its tol, normwise err, its tol)] for out, dx and every parameter gradient"""
    ref_out, ref_grads = ref
    rows = []
    for name, a, b in [("out", out, ref_out)] + [(n, grads[n], ref_grads[n]) for n in ref_grads]:
        cls = "dx" if name == "x" else tensor_class(name)
        ntol = NORM_TOL[dtype][cls]
        rows.append((name, cls, rel_err(a, b), TOL[dtype] if name == "out" else GRAD_TOL[dtype], norm_err(a, b), ntol))
    return rows


def run(c, m, x, dout, hooks=None):
    """one forward and backward of a CUDA copy of ``m`` under autocast in c.dtype: (out, {'x' | name: grad})"""
    mg = copy.deepcopy(m).cuda()
    xg = x.cuda()
    if c.layer:
        xg = xg.contiguous(memory_format=torch.channels_last_3d)
    xg.requires_grad_()
    names = [n for n, _ in mg.named_parameters()]
    params = dict(mg.named_parameters())
    for n, fn in (hooks or {}).items():
        params[n].register_hook(fn)
    with torch.autocast("cuda", dtype=c.dtype):
        out = mg(xg)
    dy = dout.cuda().to(out.dtype)
    if c.layer:
        dy = dy.contiguous(memory_format=torch.channels_last_3d)
    grads = torch.autograd.grad(out, [xg] + [params[n] for n in names], dy)
    torch.cuda.synchronize()
    return out, dict(zip(["x"] + names, grads))


def _configure(c, monkeypatch):
    from segmamba_b200 import gemm as G
    from segmamba_b200 import mamba_simple, selective_scan_cuda
    monkeypatch.setattr(G, "MODE", c.mode)
    monkeypatch.setattr(mamba_simple, "DIRECTION_STREAMS", c.streams)
    monkeypatch.setattr(selective_scan_cuda, "LOW_MEMORY_BWD", not c.stash)


def _report(rows):
    return "\n".join("  " + " ".join(str(v) if not isinstance(v, float) else f"{v:.3e}" for v in r) for r in rows)


MEASURED = []         # (case, tensor, class, max-norm err, normwise err) of every case run: the docstring's table


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_mixer_amp_vs_fp64(c, monkeypatch):
    m, x, dout, ref = _case_data(c)
    _configure(c, monkeypatch)
    rec = Recorder(monkeypatch)
    out, grads = run(c, m, x, dout)
    check_coverage(c, rec)
    calls = replay(rec.calls)
    rec.calls.clear()
    rows = end_to_end(out, grads, ref, c.dtype)
    MEASURED.extend((c.name, r[0], r[1], r[2], r[4]) for r in rows)

    bad = [r for r in calls if not r[3] <= r[4]]
    assert not bad, f"{c.name}: native calls off their fp64 replay (call, op, output, err, tol):\n" + _report(bad)
    bad = [r for r in rows if not (r[2] <= r[3] and r[4] <= r[5])]
    assert not bad, f"{c.name}: (tensor, class, max-norm err, tol, normwise err, tol):\n" + _report(bad)


# ------------------------------------------------------------------------------------------------- layer 3: sharpness
def test_replay_catches_a_dropped_k_slice(monkeypatch):
    """a split-K dt_proj weight gradient recomputed with the last K / split_k tokens of both operands zeroed fails Layer 1"""
    from segmamba_b200 import gemm as G
    c = CASES[1]
    assert c.mode == "auto" and c.L == STAGES[1][1]
    m, x, dout = _inputs(c)
    _configure(c, monkeypatch)
    rec = Recorder(monkeypatch)
    run(c, m, x, dout)
    d_inner, R8 = 2 * c.d_model, 8
    dts = [g for g in rec.of("gemm") if g.args["split_k"] > 1 and tuple(g.result.shape) == (d_inner, R8)]
    assert len(dts) == 3, "one dt_proj weight gradient per direction"
    a = dict(dts[0].args)
    ((err, tol),) = [(e, t) for _, e, t in check_gemm(a, dts[0].result)]
    assert err <= tol
    K, split_k = a["a"].shape[1], a["split_k"]
    for k in ("a", "b"):
        a[k] = a[k].clone()
        a[k][:, K - K // split_k:] = 0
    res = G.gemm(a["a"], a["b"], out_dtype=torch.float32, split_k=split_k)
    torch.cuda.synchronize()
    a["a"], a["b"] = dts[0].args["a"], dts[0].args["b"]            # compared with the product of the intact operands
    ((err, tol),) = [(e, t) for _, e, t in check_gemm(a, res)]
    assert err > tol, f"dropping 1/{split_k} of K moved the product by {err:.2e} only"


def test_end_to_end_catches_one_percent_in_one_gradient(monkeypatch):
    """dt_proj_s.weight's gradient scaled by 1.01: the normwise check fails for that parameter and for no other (in fp16, whose
    noise floor is 8x below bf16's; see the module docstring)"""
    (c,) = [c for c in CASES if c.name == "mamba-s1-f16-auto"]
    m, x, dout, ref = _case_data(c)
    _configure(c, monkeypatch)
    out, grads = run(c, m, x, dout, hooks={"dt_proj_s.weight": lambda g: g * 1.01})
    rows = end_to_end(out, grads, ref, c.dtype)
    failed = [r[0] for r in rows if r[4] > r[5]]
    assert failed == ["dt_proj_s.weight"], _report(rows)
