"""Per-phase and per-barrier-site stall breakdown of one kernel from an ncu source-page export.

    tools/sass_dump.sh                       # -> /tmp/api.sass  (nvdisasm -g of the cubin inside csrc/api.o)
    python tools/ncu_phases.py ncu_out/<name>_source.csv /tmp/api.sass <mangled-substring> [mpsa|mpfa]

Inputs: the SASS view of `ncu --page source --csv` (tools/ncu_capture.sh writes it) and the line table of
the SAME build.  Output: (1) stall-reason totals, (2) instructions / stall samples per phase of the node
routine (phase boundaries are read from the `// ---- phase N` comments of the source file), (3) barrier
stall samples grouped by the BAR.SYNC that precedes the sampled instruction -- a barrier wait is the
time the slowest warp spent in the section BEFORE that barrier, which is how low-parallelism sections
of the node routines show up."""
import collections
import csv
import os
import re
import sys

csv.field_size_limit(10**9)
src, sassf, pat = sys.argv[1], sys.argv[2], sys.argv[3]
which = sys.argv[4] if len(sys.argv) > 4 else "mpsa"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
node_file = {"mpsa": "mpsa_node.cuh", "mpfa": "node_kernels.cuh"}[which]

# phase boundaries from the source comments
bounds = []
for no, line in enumerate(open(os.path.join(ROOT, "porepy_b200", "csrc", node_file)), 1):
    m = re.search(r"// ---- phase (\w+)[ :(]", line)
    if m:
        bounds.append((no, "phase " + m.group(1)))


def phase_of(ln):
    name = "before phase 1"
    for no, nm in bounds:
        if ln >= no:
            name = nm
    return name


sass = open(sassf).read().split("\n")
start = [i for i, l in enumerate(sass) if ".text." in l and pat in l and l.strip().startswith("//---")]
if not start:
    sys.exit(f"no .text section matching {pat!r} in {sassf}")
cur, inst = None, []
for l in sass[start[0] + 1:]:
    if l.startswith("//--------------------- .text.") and inst:
        break
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        cur = (m.group(1).split("/")[-1], int(m.group(2)))
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
    if m:
        inst.append((cur, m.group(2).strip()))
rows = list(csv.reader(open(src)))
h = rows[1]
ix = {c: i for i, c in enumerate(h)}
data = rows[2:]
if len(inst) != len(data):
    sys.exit(f"SASS ({len(inst)} instructions) and ncu export ({len(data)}) are from different builds")
reasons = [c for c in h if c.startswith("stall_") and "Not Issued" not in c]
tot_s = sum(int(r[ix["# Samples"]] or 0) for r in data)
tot_i = sum(int(r[ix["Instructions Executed"]] or 0) for r in data)

by = collections.Counter()
for r in data:
    for c in reasons:
        by[c] += int(r[ix[c]] or 0)
print("stall reasons (% of samples):", {k[6:]: round(v / tot_s * 100, 1) for k, v in by.most_common(8)})


def bucket(cur):
    if cur is None:
        return "(no line info)"
    f, ln = cur
    if f == node_file and (which == "mpsa" or ln >= bounds[0][0] - 40):
        return phase_of(ln)
    if f == "node_kernels.cuh":
        return "solver / team / dmma helpers (node_kernels.cuh)"
    return f


ins, smp = collections.Counter(), collections.Counter()
for k in range(len(inst)):
    b = bucket(inst[k][0])
    ins[b] += int(data[k][ix["Instructions Executed"]] or 0)
    smp[b] += int(data[k][ix["# Samples"]] or 0)
print("\nphase / file                                         instr %  samples %")
for b in sorted(ins):
    print(f"{b:52s} {ins[b] / tot_i * 100:6.1f}  {smp[b] / tot_s * 100:8.1f}")

agg, last = collections.Counter(), None
for k in range(len(inst)):
    if inst[k][1].startswith("BAR") or " BAR." in inst[k][1]:
        last = k
    b = int(data[k][ix["stall_barrier"]] or 0)
    if b:
        agg[(last, inst[k][0])] += b
print("\nbarrier waits (% of samples) by preceding BAR (SASS index) and the line the wait is charged to")
for (lb, at), v in agg.most_common(15):
    print(f"{v / tot_s * 100:6.2f}  BAR #{lb}  -> {at}")
