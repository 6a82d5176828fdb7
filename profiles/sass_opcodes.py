"""SASS opcode summary per kernel of the shipped library (evidence that the wgmma / TMA-bulk
instructions are where DESIGN.md says they are):  python profiles/sass_opcodes.py > profiles/r02_sass_opcodes.md"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "sbi_b200", "lib", "libsbi_b200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
WANT = ["HGMMA", "UBLKCP", "UBLKRED", "SYNCS", "FFMA", "MUFU", "LDS", "STS", "LDG", "STG",
        "LDL", "STL", "BAR"]
fn, cnt, tot = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        fn = m.group(1)
        cnt[fn] = collections.Counter()
        tot[fn] = 0
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and fn:
        op = m.group(1).split(".")[0]
        tot[fn] += 1
        if op in WANT:
            cnt[fn][op] += 1
dem = subprocess.run(["cu++filt"] + list(cnt), capture_output=True, text=True).stdout.splitlines()
print("# SASS opcode counts per kernel (`cuobjdump -sass sbi_b200/lib/libsbi_b200.so`, sm_90a)\n")
print("HGMMA = wgmma.mma_async, UBLKCP = cp.async.bulk (TMA bulk copy), "
      "UBLKRED = cp.reduce.async.bulk, SYNCS = mbarrier ops, LDL / STL = local-memory (spill) traffic.\n")
print("| kernel | SASS instr | " + " | ".join(WANT) + " |")
print("|---|---|" + "---|" * len(WANT))
for (f, c), d in zip(cnt.items(), dem):
    name = re.sub(r"\(.*", "", d).replace("void ", "").replace("sbi::", "")
    print(f"| `{name}` | {tot[f]} | " + " | ".join(str(c.get(w, 0)) for w in WANT) + " |")
