"""Cost of ns_compress_bam_mapped on one aligned batch, against ns_compress_bam on the same batch, in one context with
nothing else on the device: guppy FASTQ on the 5 Mb synthetic reference, one batch of N reads (default 262 144).

- Host clock around every call (each ends in a device synchronise): the first call of each kind grows the context's
  buffers (cudaMalloc / cudaFree), the later ones reuse them.
- Then one more call of each kind under torch.profiler with CUDA activities: the device time of every kernel of the
  call (aln_count_kernel, aln_write_kernel, the deflate and pack kernels, the CUB scans), summed by name.
Prints one JSON line, with the GPU's name and power limit."""
import json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import synth
import parity_checks as pc
from nanosim_b200 import _lib as L
from nanosim_b200.records import name_table
from nanosim_b200.reference_fasta import PackedReference

n = int(sys.argv[1]) if len(sys.argv) > 1 else 262144
reps = 5
ref = PackedReference.from_records(synth.ecoli5m())
eng, _, _ = pc.make_engine("guppy", ref, fastq=True, seed=1)
info = eng.simulate(L.NS_KIND_ALIGNED, 0, n)
b = eng.fetch()
names = name_table(b, ref.names, 0)
out = {"reads": n, "bases": int(info.total_bases), "n_ops": int(info.n_ops)}
for key, fn in (("ns_compress_bam", eng.compress_bam), ("ns_compress_bam_mapped", eng.compress_bam_mapped)):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        nz = fn(names)
        t.append(time.perf_counter() - t0)
    out[key] = {"bytes": nz, "first_call_ms": round(1e3 * t[0], 2), "later_calls_ms": [round(1e3 * x, 2) for x in t[1:]]}

import torch
from torch.profiler import ProfilerActivity, profile
torch.cuda.init()
for key, fn in (("ns_compress_bam", eng.compress_bam), ("ns_compress_bam_mapped", eng.compress_bam_mapped)):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(names)
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.split("(")[0][:80]
            kern[k] = kern.get(k, 0.0) + e.device_time_total / 1e3
    out[key]["kernels_ms"] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True).stdout.strip()
eng.close()
print(json.dumps(out))
