"""Group the executed warp instructions of one kernel in an ncu report by function (source-line ranges).
usage: ncu_groups.py <report.ncu-rep> <mangled kernel name> [strict|fast]"""
import collections, csv, os, re, subprocess, sys, tempfile
rep, kern = sys.argv[1:3]
unit = sys.argv[3] if len(sys.argv) > 3 else "strict"
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tmp = tempfile.mkdtemp()
src_csv = os.path.join(tmp, "src.csv")
subprocess.run(f"ncu -i {rep} --page source --csv > {src_csv} 2>/dev/null", shell=True, check=True)
subprocess.run(f"cd {tmp} && cuobjdump -xelf svsdf_kernels_{unit} {root}/implicit_svsdf_planner_b200/lib/libsvsdf_b200.so > /dev/null 2>&1 && "
               f"nvdisasm --print-line-info svsdf_kernels_{unit}.sm_90a.cubin > sass.txt 2>/dev/null", shell=True, check=True)
# function extents from the source file
lines = open(os.path.join(root, "implicit_svsdf_planner_b200", "csrc", "svsdf_kernels.cuh")).read().split("\n")
marks = []
for i, l in enumerate(lines, 1):
    m = re.match(r"(?:static\s+)?(?:__device__|__global__)[^(]*?\b(\w+)\s*\(", l) or re.match(r"\s+(k_\w+)\(const", l)
    if m: marks.append((i, m.group(1)))
def fn_of(l):
    name = "?"
    for i, n in marks:
        if i <= l: name = n
        else: break
    return name
off2line = {}; cur = None; inside = False
for ln in open(os.path.join(tmp, "sass.txt"), errors="ignore"):
    if ln.startswith(".text." + kern): inside = True; continue
    if inside and ln.startswith("//---------------------"): break
    if not inside: continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
    if m: cur = (m.group(1).split("/")[-1], int(m.group(2))); continue
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*);", ln)
    if m: off2line[int(m.group(1), 16)] = cur
rows = list(csv.reader(open(src_csv))); hdr = rows[1]; ia = hdr.index("Instructions Executed")
base = None; grp = collections.Counter(); fp = collections.Counter(); tot = 0
for r in rows[2:]:
    try: addr = int(r[0], 16); n = int(r[ia])
    except Exception: continue
    if base is None: base = addr
    f, l = off2line.get(addr - base, ("?", 0))
    if f == "svsdf_kernels.cuh": g = fn_of(l)
    elif f == "svsdf_shapes.cuh": g = {13: "smaxd/smind", 14: "smaxd/smind", 15: "smaxd/smind", 16: "len2 (sqrt)"}.get(l, "shape functor")
    else: g = f
    grp[g] += n; tot += n
    if re.search(r"\b(DFMA|DMUL|DADD|DSETP)\b", r[1]): fp[g] += n
print(f"total warp instructions {tot}")
for g, n in grp.most_common():
    if n: print(f"{g:34s} {n/1e6:9.1f}M {100*n/tot:6.2f}%  fp64 {100*fp[g]/n:5.1f}%")
