"""Static SASS size of one kernel and of every non-inlined routine it calls (instructions without NOPs, IMAD.WIDE count, call sites).
usage: cuobjdump -sass rusty_kaspa_b200/libkgv.so > k.sass; python tools/sass_funcs.py k.sass _Z16k_schnorr_verifyILb1ELb0EEvPKhS1_S1_mPhPKjS4_S4_"""
import collections
import re
import sys

CALL = re.compile(r"CALL\.REL(?:\.NOINC)?\s+(0x[0-9a-f]+)")
path, kernel = sys.argv[1], sys.argv[2]
sec = [s for s in open(path).read().split("Function : ") if s.split("\n")[0].strip() == kernel]
assert sec, "kernel not found: " + kernel
ins = [(int(m.group(1), 16), m.group(2).strip()) for l in sec[0].split("\n") for m in [re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", l)] if m]
bounds = [0] + sorted({int(m.group(1), 16) for _, t in ins for m in [CALL.search(t)] if m}) + [1 << 62]
regions = {}
for a, b in zip(bounds, bounds[1:]):
    body = [t for addr, t in ins if a <= addr < b and not t.startswith("NOP")]
    regions[a] = (body, collections.Counter(int(m.group(1), 16) for t in body for m in [CALL.search(t)] if m))
for a, (body, calls) in regions.items():
    print("%7x  %s  instructions %5d  IMAD.WIDE %4d  call sites inside %4d  called from %3d sites" % (
        a, "kernel body" if a == 0 else "routine    ", len(body), sum("IMAD.WIDE" in t for t in body), sum(calls.values()),
        sum(c.get(a, 0) for _, c in regions.values())))
