#!/usr/bin/env python
"""summarise `nvcc -Xptxas=-v` output: per kernel stack frame, spills, registers"""
import re, subprocess, sys


def strip_params(name):
    """drop the trailing parameter list, keeping template arguments such as k_evm_group<(int)8>"""
    depth = 0
    for k in range(len(name) - 1, -1, -1):
        depth += {")": 1, "(": -1}.get(name[k], 0)
        if depth == 0:
            return name[:k] if name.endswith(")") else name
    return name


txt = open(sys.argv[1]).read()
pat = re.compile(r"Compiling entry function '([^']+)' for 'sm_90a'\nptxas info    : Function properties for \S+\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info    : Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes cumulative stack size)?")
for m in pat.finditer(txt):
    name = subprocess.run(["cu++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
    name = strip_params(name)
    print(f"{name:48s} regs={m.group(5):>3s} stack={m.group(2):>6s} cum={m.group(6) or 0:>6} spill st/ld={m.group(3)}/{m.group(4)}")
