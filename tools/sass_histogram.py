"""SASS opcode histogram of the library's kernels (what shows a Hopper-native, non-contraction kernel: UBLKCP / UBLKPF = 1-D bulk
TMA, SYNCS = mbarrier; no HMMA / HGMMA expected: there is no contraction on this path).
   python tools/sass_histogram.py acl_b200/libaclb200.so > sass_histogram.txt"""
import collections, re, subprocess, sys
lib = sys.argv[1]
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", txt)))
print("library:", lib, " architectures:", arch)
total = collections.Counter()
for block in txt.split("Function : ")[1:]:
    name = block.split("\n", 1)[0]
    ops = collections.Counter()
    for line in block.split("\n"):
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m:
            ops[m.group(1)] += 1
    total.update(ops)
    short = re.sub(r"_ZN7aclb200\d+_GLOBAL__N__\w+?_cu_\w{8}\d+", "", name)
    if "pipeline_kernelILi1ELb0ELb0E" in name or "scalar_tracks_pipeline_kernelILi1ELb0" in name or "build_base" in name:
        print(f"\n{short[:100]}: {sum(ops.values())} instructions")
        print("  " + ", ".join(f"{k} {v}" for k, v in ops.most_common(28)))
print("\nwhole library:", sum(total.values()), "instructions")
for key in ("UBLKCP", "UBLKPF", "SYNCS", "UTMACMDFLUSH", "ATOMS", "HMMA", "HGMMA", "LDGSTS"):
    print(f"  {key:14s} {total.get(key, 0)}")
