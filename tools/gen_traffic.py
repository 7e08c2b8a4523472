#!/usr/bin/env python
"""Generator DRAM traffic of one infer() step from an ncu launch list (tools/profile_step.py under
`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum`): sums dram__bytes over the launches of the LAST
step's Generator stage (k_c4_to_h8 .. k_conv_post_tanh*) and writes profiles/<tag>_generator_traffic.json stamped with the build id
of the CUDA sources, which bench.py requires to match before it reports `roofline.traffic`."""
import argparse, collections, csv, json, os, re, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("csv"); ap.add_argument("out"); ap.add_argument("--frames", type=int, required=True); ap.add_argument("--precision", default="fp16")
a = ap.parse_args()
rows = [r for r in csv.reader(l for l in open(a.csv) if l.startswith('"'))]
hdr = rows[0]; idx = {h: i for i, h in enumerate(hdr)}
per = collections.OrderedDict()
for r in rows[1:]:
    if len(r) < len(hdr): continue
    lid = int(r[idx["ID"]])
    d = per.setdefault(lid, {"name": re.sub(r"\(.*$", "", re.sub(r"^void\s+", "", r[idx["Kernel Name"]])).replace("bv2::", ""), "us": 0.0, "bytes": 0.0})
    v = float(r[idx["Metric Value"]].replace(",", "")); u = r[idx["Metric Unit"]]; m = r[idx["Metric Name"]]
    if m.startswith("gpu__time"): d["us"] = v * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1.0)
    elif m.startswith("dram__bytes"): d["bytes"] += v * {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1.0)
ids = list(per)
ends = [i for i in ids if per[i]["name"].startswith("k_conv_post_tanh")]
starts = [i for i in ids if per[i]["name"].startswith("k_c4_to_h8")]
end = ends[-1]
start = max(i for i in starts if i < end and not any(e < end and e > i for e in ends))
first = min(i for i in starts if i <= start and i > ([e for e in ends if e < end] or [-1])[-1])
gen = [i for i in ids if first <= i <= end]
tot = sum(per[i]["bytes"] for i in gen)
import bench
out = {"frames": a.frames, "generator_dram_bytes": tot, "generator_dram_bytes_per_frame": tot / a.frames, "generator_launches": len(gen),
       "generator_us_serialised": sum(per[i]["us"] for i in gen), "build_id": bench.build_id(), "generator_build_id": bench.generator_build_id(),
       "source": f"ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum ({os.path.basename(a.csv)}), config 2, {a.precision} engine, last captured step"}
json.dump(out, open(a.out, "w"), indent=1)
print(json.dumps(out))
