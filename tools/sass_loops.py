"""Static instruction mix of the loops of a kernel from `cuobjdump -sass` (no GPU needed).

usage: python tools/sass_loops.py <lib.so> <mangled-kernel-substring> [min_len]
For every backward branch (loop) prints the body length and the opcode histogram, so the instructions per scan update can
be counted before spending GPU time.
"""
import collections
import re
import subprocess
import sys


def disasm(lib, pattern):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    out, cur, name = {}, None, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            cur = out.setdefault(name, [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2).strip()))
    return {k: v for k, v in out.items() if pattern in k}


def opcode(ins):
    ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
    return ins.split()[0]


def main():
    lib, pat = sys.argv[1], sys.argv[2]
    min_len = int(sys.argv[3]) if len(sys.argv) > 3 else 40
    for name, code in disasm(lib, pat).items():
        print("==", name, len(code), "instructions")
        addr_index = {a: i for i, (a, _) in enumerate(code)}
        for i, (a, ins) in enumerate(code):
            m = re.search(r"BRA(?:\.\w+)*\s+(?:!?U?P\d+,\s*)?(0x[0-9a-f]+)", ins)
            if not m:
                continue
            tgt = int(m.group(1), 16)
            if tgt >= a or tgt not in addr_index:
                continue
            body = code[addr_index[tgt]:i + 1]
            if len(body) < min_len:
                continue
            hist = collections.Counter(opcode(x).split(".")[0] for _, x in body)
            full = collections.Counter(opcode(x) for _, x in body)
            print(f"  loop 0x{tgt:x}..0x{a:x}: {len(body)} instr; MUFU.EX2 {full.get('MUFU.EX2', 0)}, MUFU.RCP {full.get('MUFU.RCP', 0)}")
            print("    " + ", ".join(f"{k} {v}" for k, v in hist.most_common(18)))


if __name__ == "__main__":
    main()
