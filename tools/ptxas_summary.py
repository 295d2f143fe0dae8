#!/usr/bin/env python
"""summarise `nvcc -Xptxas=-v` output: per kernel stack frame, spills, registers"""
import re, subprocess, sys
txt = open(sys.argv[1]).read()
pat = re.compile(r"Compiling entry function '([^']+)' for 'sm_90a'\nptxas info    : Function properties for \S+\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info    : Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes cumulative stack size)?")
for m in pat.finditer(txt):
    name = subprocess.run(["cu++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
    name = re.sub(r"\(.*", "", name)
    print(f"{name:48s} regs={m.group(5):>3s} stack={m.group(2):>6s} cum={m.group(6) or 0:>6} spill st/ld={m.group(3)}/{m.group(4)}")
