"""Cost of NM and SA (ns_set_aln_tags) in ns_compress_bam_mapped: guppy FASTQ on the 5 Mb synthetic reference, one batch
of N reads (default 262 144), simulated alike (same seed) in two contexts, one of them with the tags' tables.

- Host clock around every call (each ends in a device synchronise), the two contexts alternated; the first call of each
  grows its buffers, the later ones reuse them.
- Then one more call of each under torch.profiler with CUDA activities: the device time of every kernel, summed by name.
Prints one JSON line, with the GPU's name and power limit."""
import json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth
import parity_checks as pc
from nanosim_b200 import _lib as L
from nanosim_b200.records import name_table
from nanosim_b200.reference_fasta import PackedReference

n = int(sys.argv[1]) if len(sys.argv) > 1 else 262144
reps = 7
ref = PackedReference.from_records(synth.ecoli5m())
arms = {}
for key in ("untagged", "tagged"):
    eng, _, _ = pc.make_engine("guppy", ref, fastq=True, seed=1)
    if key == "tagged":
        eng.set_aln_tags(list(ref.raw_names))
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, n)
    arms[key] = (eng, name_table(eng.fetch(), ref.names, 0))
out = {"reads": n, "bases": int(info.total_bases), "n_ops": int(info.n_ops)}
t = {k: [] for k in arms}
nbytes = {}
for _ in range(reps):
    for key, (eng, names) in arms.items():
        t0 = time.perf_counter()
        nbytes[key] = eng.compress_bam_mapped(names)
        t[key].append(time.perf_counter() - t0)
for key in arms:
    out[key] = {"bytes": nbytes[key], "first_call_ms": round(1e3 * t[key][0], 2),
                "later_calls_ms": [round(1e3 * x, 2) for x in t[key][1:]]}

import torch
from torch.profiler import ProfilerActivity, profile
torch.cuda.init()
for key, (eng, names) in arms.items():
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.compress_bam_mapped(names)
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.split("(")[0][:80]
            kern[k] = kern.get(k, 0.0) + e.device_time_total / 1e3
    out[key]["kernels_ms"] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True).stdout.strip()
for eng, _ in arms.values():
    eng.close()
print(json.dumps(out))
