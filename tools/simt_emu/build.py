"""Build the CPU-emulated twin of libsegmamba_b200.so: the SAME kernel sources, run by tools/simt_emu (fibers instead of CUDA
threads).  TEST INFRASTRUCTURE ONLY -- the product never loads this library.

    python tools/simt_emu/build.py          ->  tools/simt_emu/_build/libsegmamba_b200_emu.so

The .cu files are used as they are, except for two constructs that are CUDA syntax rather than C++ and are rewritten
textually into tools/simt_emu/_build/gen/*.cpp:

    kernel<targs><<<grid, block, smem, stream>>>(args);   ->  SMB_EMU_LAUNCH((kernel<targs>), grid, block, smem, args);
    extern __shared__ [__align__(16)] float name[];        ->  float *name = (float *)emu::dyn_smem();

Inline PTX sits behind `#ifdef SMB_EMU` in csrc/common.cuh (ex2, prefetch, vector red).
"""
from __future__ import annotations

import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "segmamba_b200", "csrc")
BUILD = os.path.join(HERE, "_build")
OUT = os.path.join(BUILD, "libsegmamba_b200_emu.so")
SOURCES = ["capi.cu", "scan_fwd.cu", "scan_fwd_v2.cu", "scan_bwd.cu", "scan_bwd_v2.cu", "scan_bwd_r3v2.cu", "conv1d.cu", "conv1d_v2.cu", "instnorm.cu", "layernorm.cu", "layout.cu", "augment.cu", "metrics.cu", "predict.cu", "preprocess.cu"]
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"


def _match_back_template(text: str, end: int) -> int:
    """text[end-1] == '>' closes a template argument list; return the index of its '<'."""
    depth = 0
    i = end - 1
    while i >= 0:
        if text[i] == ">":
            depth += 1
        elif text[i] == "<":
            depth -= 1
            if depth == 0:
                return i
        i -= 1
    raise ValueError("unbalanced template brackets before <<<")


def _match_paren(text: str, start: int) -> int:
    """text[start] == '('; return the index of the matching ')'."""
    depth = 0
    for i in range(start, len(text)):
        if text[i] == "(":
            depth += 1
        elif text[i] == ")":
            depth -= 1
            if depth == 0:
                return i
    raise ValueError("unbalanced parentheses in a kernel launch")


def rewrite_launches(text: str) -> str:
    out = []
    pos = 0
    while True:
        k = text.find("<<<", pos)
        if k < 0:
            out.append(text[pos:])
            return "".join(out)
        # kernel expression: identifier [ <template args> ] immediately before <<<
        e = k
        while text[e - 1].isspace():
            e -= 1
        s = e
        if text[s - 1] == ">":
            s = _match_back_template(text, s)
        while s > 0 and (text[s - 1].isalnum() or text[s - 1] in "_:"):
            s -= 1
        kernel = text[s:e]
        c_end = text.find(">>>", k)
        config = text[k + 3:c_end]
        a_start = c_end + 3
        while text[a_start].isspace():
            a_start += 1
        assert text[a_start] == "(", f"no argument list after the launch of {kernel}"
        a_end = _match_paren(text, a_start)
        args = text[a_start + 1:a_end]
        # config = grid, block, smem, stream  (split on top-level commas)
        parts, depth, cur = [], 0, ""
        for ch in config:
            if ch in "([":
                depth += 1
            elif ch in ")]":
                depth -= 1
            if ch == "," and depth == 0:
                parts.append(cur.strip())
                cur = ""
            else:
                cur += ch
        parts.append(cur.strip())
        while len(parts) < 3:
            parts.append("0")
        grid, block, smem = parts[0], parts[1], parts[2]
        out.append(text[pos:s])
        out.append(f"SMB_EMU_LAUNCH(({kernel}), {grid}, {block}, {smem}, {args})")
        pos = a_end + 1


_EXTERN_SHARED = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?(\w+)\s+(\w+)\[\];")


def transform(text: str) -> str:
    text = _EXTERN_SHARED.sub(lambda m: f"{m.group(1)} *{m.group(2)} = reinterpret_cast<{m.group(1)} *>(emu::dyn_smem());", text)
    return rewrite_launches(text)


def build(verbose: bool = False, opt: str = "-O1", asan: bool = False) -> str:
    """asan=True: AddressSanitizer build (libsegmamba_b200_emu_asan.so) -- out-of-bounds reads / writes of any kernel on the
    (host) tensors abort with a report; run python with LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0."""
    global OUT
    if asan:
        OUT = os.path.join(BUILD, "libsegmamba_b200_emu_asan.so")
    gen = os.path.join(BUILD, "gen_asan" if asan else "gen")
    os.makedirs(gen, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    deps += [os.path.join(HERE, f) for f in ("simt_emu.h", "simt_emu.cpp", "build.py")] + [os.path.join(ROOT, "include", "segmamba_b200.h")]
    if os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in deps):
        return OUT
    cpps = []
    for name in SOURCES:
        src = open(os.path.join(CSRC, name)).read()
        dst = os.path.join(gen, name.replace(".cu", "_emu.cpp"))
        with open(dst, "w") as f:
            f.write(f'// GENERATED by tools/simt_emu/build.py from segmamba_b200/csrc/{name} -- do not edit\n#include "simt_emu.h"\n')
            f.write(f'#line 1 "{os.path.join(CSRC, name)}"\n')
            f.write(transform(src))
        cpps.append(dst)
    cpps.append(os.path.join(HERE, "simt_emu.cpp"))
    flags = ["-std=c++17", opt, "-g", "-fPIC", "-DSMB_EMU=1", "-fno-strict-aliasing", "-w", "-I", HERE, "-I", CSRC, "-I", CUDA_INC]
    if asan:
        flags += ["-fsanitize=address", "-fno-omit-frame-pointer"]
    env = dict(os.environ)
    env.pop("LD_PRELOAD", None)                                  # a preloaded libasan (memcheck runs) must not instrument the compiler
    procs, objs = [], []
    for cpp in cpps:                                             # one compiler process per translation unit, in parallel
        obj = os.path.join(gen, os.path.basename(cpp)[:-4] + ".o")
        cmd = ["/usr/bin/g++"] + flags + ["-c", cpp, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((cmd, subprocess.Popen(cmd, env=env)))
        objs.append(obj)
    for cmd, p in procs:
        if p.wait() != 0:
            raise subprocess.CalledProcessError(p.returncode, cmd)
    # -Bsymbolic: the stubbed CUDA runtime entry points must bind inside this library even when a real libcudart is loaded
    subprocess.run(["/usr/bin/g++", "-shared", "-o", OUT] + objs + ["-lpthread", "-Wl,-Bsymbolic"] + (["-fsanitize=address"] if asan else []),
                   check=True, env=env)
    return OUT


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if a != "--asan"]
    print(build(verbose=True, opt=args[0] if args else "-O1", asan="--asan" in sys.argv))
