"""DRAM traffic of the dominant kernel from an `ncu --set full` capture -> profiles/traffic_<workload>.json, which bench.py
puts into roofline.traffic (bytes per launch: dram__bytes_read.sum + dram__bytes_write.sum).

    python tools/ncu_traffic.py profiles/emit.ncu-rep config2 emit_kernel "<command the capture was taken with>"
"""
import csv
import json
import os
import subprocess
import sys

rep, workload, kernel = sys.argv[1], sys.argv[2], sys.argv[3]
cmd = sys.argv[4] if len(sys.argv) > 4 else ""
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
out = None
for vals in rows[2:]:
    if kernel not in vals[hdr.index("Kernel Name")]:
        continue

    def get(name):
        i = hdr.index(name)
        v = float(vals[i].replace(",", ""))
        u = units[i].lower()
        return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[u]

    rd, wr = get("dram__bytes_read.sum"), get("dram__bytes_write.sum")
    out = {"workload": workload, "kernel": vals[hdr.index("Kernel Name")], "dram_bytes_read": rd, "dram_bytes_write": wr,
           "dram_bytes_per_launch": rd + wr, "duration_ms_under_ncu": float(vals[hdr.index("gpu__time_duration.sum")].replace(",", "")) *
           {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3}[units[hdr.index("gpu__time_duration.sum")]],
           "source": "ncu --set full capture %s (%s)" % (os.path.basename(rep), cmd or "see profiles/")}
    break
assert out, "kernel not found in the report"
path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "traffic_%s.json" % workload)
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(path, out["dram_bytes_per_launch"] / 1e9, "GB per launch")
