"""Cost of the emit kernel on config 2 in one context: the guppy FASTQ model on the 3.09 Gb synthetic hg38-sized reference
(bench.py's config 2), its aligned batch (235 536 reads) and its unaligned batch (26 608 reads), each with fresh read ids.

- Per batch kind, after three warm-up batches, `--batches` (default 10) batches are timed by the library's own CUDA
  events: ``ms_emit`` spans emit_kernel (it starts after split_kernel), ``ms_total`` the whole batch.
- Then three more batches of each kind under torch.profiler with CUDA activities: the device time of every kernel,
  summed by name and divided by the batch count.
Prints one JSON line, with the GPU's name, power limit and clocks.  NANOSIM_B200_LIB selects another build of the library."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
from nanosim_b200 import _lib as L
from nanosim_b200.engine import Engine
from nanosim_b200.model import CompiledModel, DeviceTables

ap = argparse.ArgumentParser()
ap.add_argument("--batches", type=int, default=10)
ap.add_argument("--label", default="")
args = ap.parse_args()

import torch
torch.cuda.set_device(0)
W = bench.WORKLOADS["config2"]
sref = bench.build_reference("config2", 0, 1.0, True)
n_bases = int(sref.offsets[-1])
tables = DeviceTables(CompiledModel.load(os.path.join(bench.DATA, W["model"])), fastq=True, chimeric=False, homopolymer=False,
                      mode="genome")
eng = Engine(device=0, seed=20260924)
eng.set_reference_ptr(sref.bases.data_ptr(), n_bases, sref.offsets)
eng.set_model(tables)
eng.configure(fastq=True, min_len=50, max_len=sref.max_chrom)
n_al, n_un = tables.split_counts(W["batch"])
BATCH = {"aligned": (L.NS_KIND_ALIGNED, n_al), "unaligned": (L.NS_KIND_UNALIGNED, n_un)}
batch = {"aligned": 0, "unaligned": 0}


def run(name):
    kind, n = BATCH[name]
    info = eng.simulate(kind, batch[name] * n, n)
    batch[name] += 1
    return info


def mean(xs):
    return round(sum(xs) / len(xs), 3)


out = {"label": args.label, "lib": os.path.basename(L.LIB_PATH)}
for name in BATCH:
    for _ in range(3):
        run(name)
    rows = [run(name) for _ in range(args.batches)]
    emit = [r.ms_emit for r in rows]
    out[name] = {"reads": BATCH[name][1], "bases_per_batch": mean([r.total_bases for r in rows]),
                 "ms_emit": [round(x, 3) for x in emit], "ms_emit_mean": mean(emit), "ms_emit_min": round(min(emit), 3),
                 "ms_plan_mean": mean([r.ms_plan for r in rows]), "ms_total_mean": mean([r.ms_total for r in rows])}

from torch.profiler import ProfilerActivity, profile
n_prof = 3
for name in BATCH:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            run(name)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.split("(")[0][:80]
            kern[k] = kern.get(k, 0.0) + e.device_time_total / 1e3 / n_prof
    out[name]["kernels_ms_per_batch"] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])[:8]}
out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip()
eng.close()
print(json.dumps(out), flush=True)
