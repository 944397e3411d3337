#!/usr/bin/env python
"""Memory instructions of ctu_frame_kernel per device function, from the SASS of a build: generic LD / ST (the L1TEX
path, whatever the address space), shared LDS / STS, local LDL / STL (the thread's stack: by-reference arguments, local
arrays, spills), instructions and code bytes.  Static counts, not executed ones.

    python tools/sass_census.py kvazaar_b200/libkvzcuda.so [function ...]     # one markdown table per instantiation
"""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ncu_ctu_summary import function_of_each_instruction  # noqa: E402

KINDS = ("LD", "ST", "LDS", "STS", "LDL", "STL")
INSN_BYTES = 16           # every sm_90 instruction is 128 bits
PIX = {"h": "uint8_t", "t": "uint16_t"}


def opcode(line):
    """Mnemonic of one nvdisasm line, without predicate and modifiers ("@!P0 LD.E.64 R2, [R4] ;" -> "LD")."""
    body = re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", line)
    body = re.sub(r"^@!?U?P[T0-9]+\s+", "", body)
    tok = body.split()
    return tok[0].split(".")[0] if tok else ""


def census(lib):
    """{instantiation: {function: {kind: count, "insn": n}}} for both instantiations of ctu_frame_kernel in `lib`."""
    out = {}
    for kern, fn, line in function_of_each_instruction(lib, with_text=True):
        c = out.setdefault(kern, {}).setdefault(fn, dict(insn=0, **{k: 0 for k in KINDS}))
        c["insn"] += 1
        op = opcode(line)
        if op in c:
            c[op] += 1
    return out


def main():
    lib = sys.argv[1]
    only = sys.argv[2:]
    for kern, fns in sorted(census(lib).items()):
        total = sum(c["insn"] for c in fns.values())
        print(f"\n## ctu_frame_kernel<{PIX.get(kern, kern)}>: {total} instructions, {total * INSN_BYTES} B of code\n")
        print("| function | LD / ST | LDS / STS | LDL / STL | instructions | bytes |\n|---|---|---|---|---|---|")
        rows = sorted(fns.items(), key=lambda kv: -kv[1]["insn"])
        if only:
            rows = [r for r in rows if any(r[0].startswith(o) for o in only)]
        for fn, c in rows:
            print(f"| {fn} | {c['LD']} / {c['ST']} | {c['LDS']} / {c['STS']} | {c['LDL']} / {c['STL']} | {c['insn']} | {c['insn'] * INSN_BYTES} |")
        s = {k: sum(c[k] for c in fns.values()) for k in KINDS}
        print(f"| (all) | {s['LD']} / {s['ST']} | {s['LDS']} / {s['STS']} | {s['LDL']} / {s['STL']} | {total} | {total * INSN_BYTES} |")


if __name__ == "__main__":
    main()
