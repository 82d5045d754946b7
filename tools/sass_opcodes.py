"""Opcode histogram per kernel of librr_b200.so (cuobjdump -sass): the SASS evidence for tcgen05 (UTCHMMA / UTCQMMA),
TMEM (LDTM / STTM), TMA (UTMALDG / UTMAPF / UTMASTG), mbarrier (SYNCS), legacy tensor ops (HMMA) and the memory
instructions of each kernel.  No GPU needed.   python tools/sass_opcodes.py > profiles/r02_sass_opcodes.txt"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "sample-resilient-llm-inference_b200", "librr_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
KEY = ["UTCHMMA", "UTCQMMA", "UTCBAR", "LDTM", "STTM", "UTMALDG", "UTMAPF", "UTMASTG", "UTMACCTL", "SYNCS", "HMMA", "LDSM", "MOVM",
       "LDG", "STG", "LDS", "STS", "ATOMG", "RED", "MEMBAR", "CCTL", "ELECT", "ACQBULK", "BAR", "MUFU", "SHFL"]
kern, hist = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        kern = m.group(1); hist[kern] = collections.Counter(); continue
    m = re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)", line)
    if m and kern:
        op, mods = m.group(1), m.group(2)
        hist[kern][op] += 1
        if op in ("UTCHMMA", "UTMALDG", "HMMA", "LDTM", "STTM") and mods:
            hist[kern][op + mods] += 1
def demangle(n):
    r = subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    r = r.replace("(anonymous namespace)::", "")
    return re.sub(r"\(.*", "", r)[:110]
print(f"# {os.path.relpath(lib, ROOT)}: {len(hist)} kernels (sm_90a SASS); columns = instruction counts")
for k, h in hist.items():
    tot = sum(v for o, v in h.items() if "." not in o)
    keys = [(o, h[o]) for o in KEY if h.get(o)]
    mods = sorted((o, v) for o, v in h.items() if "." in o)
    print(f"\n{demangle(k)}\n  total {tot}: " + ", ".join(f"{o} {v}" for o, v in keys))
    if mods:
        print("  variants: " + ", ".join(f"{o} {v}" for o, v in mods))
