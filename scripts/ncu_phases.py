"""Instruction / stall-sample share per K1 phase.  usage: python scripts/ncu_phases.py <report.ncu-rep>
Phases are found by source file + the marker comments in query.cu."""
import csv, subprocess, sys, re
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass,cuda"],
                     capture_output=True, text=True).stdout
src = open("pin_slam_b200/csrc/query.cu").read().splitlines()
def line_of(pat, start=0):
    for i in range(start, len(src)):
        if pat in src[i]:
            return i + 1
    raise SystemExit("marker not found: " + pat)
marks = [("prologue", 1), ("A1 probe loop", line_of("knn_search_lane(const")), ("neighbour_vec", line_of("__device__ __forceinline__ void neighbour_vec")),
         ("A2 gather_weighted", line_of("void gather_weighted(")), ("A2 gather_rows", line_of("void gather_rows(")),
         ("C1 group_reduce8", line_of("void group_reduce8(")), ("C1 feature_dots", line_of("void feature_dots(")),
         ("kernel prologue", line_of("void __launch_bounds__(WPB * 32, 1) query_kernel")),
         ("A1 query load / setup", line_of("phase A1: thread per query")), ("A1 winners re-read", line_of("re-read the winners")),
         ("A1 weights / vectors / stash / outputs", line_of("normalised inverse-distance weights, summed")),
         ("A2 call + wf0 rows", line_of("phase A2:")), ("B decoder glue (query.cu)", line_of("phase B: decoder")),
         ("C2 chain rule + outputs", line_of("C1: a_k = <g_xbar")), ("other kernels", line_of("search-only kernels"))]
def phase_of(f, ln):
    if f == "knn_select.cuh": return "A1 sorting networks"
    if f == "mlp_chain.cuh": return "B decoder MMA (mlp_chain.cuh)"
    if f == "common.cuh": return "A1 hash / misc (common.cuh)"
    if f != "query.cu": return "intrinsics / other headers"
    name = marks[0][0]
    for n, l in marks:
        if ln >= l: name = n
    return name
rows = list(csv.reader(out.splitlines()))
cur = None; hdr = None; agg = {}
for r in rows:
    if len(r) == 2 and r[0] == "File Path": cur = r[1].split("/")[-1]; continue
    if r and r[0] == "Line No": hdr = r; continue
    if hdr is None or len(r) != len(hdr) or r[0] == "": continue
    d = dict(zip(hdr, r))
    ph = phase_of(cur, int(r[0]))
    a = agg.setdefault(ph, [0, 0, 0])
    a[0] += int(d["# Samples"] or 0); a[1] += int(d["Instructions Executed"] or 0)
    a[2] += int(d.get("L2 Theoretical Sectors Global") or 0)
ts = sum(a[0] for a in agg.values()); ti = sum(a[1] for a in agg.values())
print("phase,stall_samples_pct,instructions_pct,warp_instructions,l2_sectors_global")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    print(f"{k},{100*a[0]/ts:.1f},{100*a[1]/ti:.1f},{a[1]},{a[2]}")
