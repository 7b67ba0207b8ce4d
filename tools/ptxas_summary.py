"""Summarise registers / spills per kernel from mpyc_b200/csrc/_obj/ptxas.log (build with -v)."""
import re, subprocess, sys
log = open('mpyc_b200/csrc/_obj/ptxas.log').read()
ents = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n.*?Used (\d+) registers", log, re.S)
names = subprocess.run(['cu++filt'] + [e[0] for e in ents], capture_output=True, text=True).stdout.split('\n')
pat = sys.argv[1] if len(sys.argv) > 1 else ''
for e, nm in zip(ents, names):
    nm = nm.replace('void ', '')
    nm = nm[:nm.index('>(') + 1] if '>(' in nm else nm[:nm.index('(')]
    if re.search(pat, nm):
        print(f"{nm:50s} regs={e[4]:>3s} stack={e[1]} spill={e[2]}/{e[3]}")
