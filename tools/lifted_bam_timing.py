"""Cost of --lift_mapped_bam at config 2's scale: tools/haplotype_build.py's genome (3.09 Gb) and ~4 M small variants
(--sv N: also about N structural variants), the haplotypes built in HBM, and one aligned guppy FASTQ batch of N reads
(default 262 144) simulated from them.  Two contexts hold the same haplotypes and simulate the same batch (same seed);
only the second keeps a lift (ns_set_lift); with --tags both keep it and only the second also has NM and SA
(ns_set_aln_tags).  Prints one JSON line:
  set_lift_ms      host clock around ns_set_lift (it ends in a device synchronise): checks, uploads, segments, scan, table
  lift_bytes       the device bytes the lift keeps
  calls_ms         host clock around ns_compress_bam_mapped, arms alternated on reused buffers (after one call each that
                   grows them)
  kernels_ms       per arm, one more call under torch.profiler with CUDA activities: device time by kernel name
  gpu              name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import parity_checks as pc  # noqa: E402
from haplotype_build import genome, sv_spans, write_vcf  # noqa: E402
from nanosim_b200 import _lib as L  # noqa: E402
from nanosim_b200.records import name_table  # noqa: E402
from nanosim_b200.variants import read_vcf  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reads", type=int, default=262144)
    ap.add_argument("--variants", type=int, default=4_000_000)
    ap.add_argument("--sv", type=int, default=0)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    ap.add_argument("--tags", action="store_true", help="time lifted records without and with NM and SA (ns_set_aln_tags) "
                    "instead of unlifted against lifted")
    args = ap.parse_args()
    ref = genome(args.scale)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.vcf")
        write_vcf(path, ref, args.variants, svs=sv_spans(ref, args.sv) if args.sv else None)
        tables = read_vcf(path, ref)
    res = {"reads": args.reads, "variants": int(tables.applied.sum()), "sv": int(tables.structural.sum()),
           "segments": 2 * len(tables.var_pos) + len(tables.hap_chrom)}
    engines = []
    keys = ("lifted", "lifted_tagged") if args.tags else ("mapped", "lifted")
    for key in keys:
        eng, _, _ = pc.make_engine("guppy", ref, fastq=True, seed=1)
        eng.apply_variants(tables)
        eng.configure(fastq=True, min_len=50, max_len=int(max(tables.lengths)))
        if key != "mapped":
            t0 = time.perf_counter()
            res["lift_bytes"] = eng.set_lift(tables)
            res["set_lift_ms"] = round(1e3 * (time.perf_counter() - t0), 2)
        if key == "lifted_tagged":
            res["tags_bytes"] = eng.set_aln_tags(list(ref.raw_names), tables.ref_paired, len(tables.var_pos))
        info = eng.simulate(L.NS_KIND_ALIGNED, 0, args.reads)
        engines.append(eng)
    res["bases"], res["n_ops"] = int(info.total_bases), int(info.n_ops)
    names = name_table(engines[0].fetch(), tables.names, 0)
    sizes = [e.compress_bam_mapped(names) for e in engines]                  # grows each context's buffers
    res["bytes"] = dict(zip(keys, sizes))
    calls = {k: [] for k in keys}
    for _ in range(args.reps):
        for key, e in zip(keys, engines):
            t0 = time.perf_counter()
            e.compress_bam_mapped(names)
            calls[key].append(round(1e3 * (time.perf_counter() - t0), 2))
    res["calls_ms"] = calls

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    res["kernels_ms"] = {}
    for key, e in zip(keys, engines):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.compress_bam_mapped(names)
        kern = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = ev.name.split("(")[0][:80]
                kern[k] = kern.get(k, 0.0) + ev.device_time_total / 1e3
        res["kernels_ms"][key] = {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
    for e in engines:
        e.close()
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                text=True).stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
