"""genome --vcf at config 2's scale: a 3.09 Gb synthetic genome (hg38 chromosome lengths, i.i.d. ACGT, as bench.py builds
it) and a synthetic VCF of about 4 M variants on it (SNVs, deletions and insertions of up to 10 and 20 bases, GT 0|1,
1|0 or 1|1).  Prints one JSON line:
  parse_s          host time of variants.read_vcf (read, parse, check, tables)
  call_ms          the whole ns_apply_variants call between CUDA events (it ends in a device synchronise): host checks of
                   the tables, their upload, segments, scan, gather, and ns_set_reference on the haplotypes
  kernel_ms        device time of each of the build's kernels, from torch.profiler in a second build of its own
  hap_bytes, gather_GBps    bytes of the haplotypes, and 2 x that (read + write) over hap_gather_kernel's time
  accounted_peak_bytes      the sizes of the library's allocations at the build's peak (ns_apply_variants' count, not a
                   device reading)
  gpu, power_limit read in the same run.
--parse-only: the host half only (no GPU needed)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synth  # noqa: E402
from nanosim_b200.reference_fasta import PackedReference  # noqa: E402
from nanosim_b200.variants import read_vcf  # noqa: E402


def genome(scale):
    rng = np.random.default_rng(1)
    lengths = [max(1000, int(x * scale)) for x in synth.HG38_LENGTHS]
    bases = np.concatenate([synth.synth_chrom(rng, n) for n in lengths])
    return PackedReference(synth.HG38_NAMES, bases, np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64))


def write_vcf(path, ref, n_variants, seed=7):
    rng = np.random.default_rng(seed)
    acgt = np.array(list("ACGT"))
    L = ref.lengths
    lines = ["##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tHG\n"]
    for c, name in enumerate(ref.names):
        n = int(n_variants * L[c] / L.sum())
        gap = max(24, int(L[c] // max(n, 1)))
        pos = np.arange(1, n + 1, dtype=np.int64) * gap - rng.integers(0, gap - 12, n)      # spans never overlap
        pos = pos[pos + 12 < L[c]]
        kind = rng.choice(3, len(pos), p=[0.8, 0.1, 0.1])
        rlen = np.where(kind == 1, rng.integers(2, 11, len(pos)), 1)
        base = int(ref.offsets[c])
        refs = [ref.bases[base + p - 1:base + p - 1 + n].tobytes().decode() for p, n in zip(pos.tolist(), rlen.tolist())]
        ins = ["".join(acgt[rng.integers(0, 4, k)]) for k in rng.integers(1, 20, len(pos)).tolist()]
        snv = acgt[rng.integers(0, 4, len(pos))]
        gts = np.array(["0|1", "1|0", "1|1"])[rng.choice(3, len(pos), p=[0.4, 0.4, 0.2])]
        for p, r, k, s, i, g in zip(pos.tolist(), refs, kind.tolist(), snv.tolist(), ins, gts.tolist()):
            alt = (s if s != r[0] else "A" if r[0] != "A" else "C") if k == 0 else r[0] if k == 1 else r[0] + i
            lines.append("%s\t%d\t.\t%s\t%s\t50\tPASS\t.\tGT\t%s\n" % (name, p, r, alt, g))
    with open(path, "w") as f:
        f.writelines(lines)
    return len(lines) - 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--variants", type=int, default=4_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="chromosome lengths x scale (1.0 = 3.09 Gb)")
    ap.add_argument("--parse-only", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()
    ref = genome(args.scale)
    res = {"genome_bases": ref.genome_len}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.vcf")
        res["vcf_records"] = write_vcf(path, ref, args.variants)
        res["vcf_bytes"] = os.path.getsize(path)
        t0 = time.perf_counter()
        tables = read_vcf(path, ref)
        res["parse_s"] = round(time.perf_counter() - t0, 3)
    res["applied"] = int(tables.applied.sum())
    res["hap_bytes"] = int(tables.offsets[-1])
    if not args.parse_only:
        import torch

        from nanosim_b200.engine import Engine
        eng = Engine(device=0, seed=1)
        eng.set_reference(ref)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        res["accounted_peak_bytes"] = eng.apply_variants(tables)
        ev[1].record()
        torch.cuda.synchronize()
        res["call_ms"] = round(ev[0].elapsed_time(ev[1]), 2)
        # spot check: the first 1 MB of every haplotype record against the tables, spliced on the host
        got = eng.reference_bases(res["hap_bytes"])
        offs = tables.offsets.astype(np.int64)
        for h, c in enumerate(tables.hap_chrom):
            seq = ref.bases[int(ref.offsets[c]):int(ref.offsets[c + 1])]
            parts, prev = [], 0
            for j in range(int(tables.var_off[h]), int(tables.var_off[h + 1])):
                if prev > 1 << 20:
                    break
                p = int(tables.var_pos[j])
                parts += [seq[prev:p], tables.alt[int(tables.alt_off[j]):int(tables.alt_off[j] + tables.alt_len[j])]]
                prev = p + int(tables.var_ref_len[j])
            parts.append(seq[prev:prev + (1 << 20)])
            want = np.concatenate(parts)[:1 << 20]
            assert np.array_equal(got[offs[h]:offs[h] + len(want)], want), tables.names[h]
        res["spot_check"] = "ok"
        eng.close()
        # the kernels' own device time, in a second build traced by torch.profiler
        from torch.profiler import ProfilerActivity, profile
        eng = Engine(device=0, seed=1)
        eng.set_reference(ref)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.apply_variants(tables)
            torch.cuda.synchronize()
        kernel_ms = {}
        for e in prof.key_averages():
            if e.key.startswith(("hap_", "pack_reference_kernel")) or "DeviceScan" in e.key:
                name = e.key.split("(")[0] if e.key.startswith(("hap_", "pack_")) else "cub_scan"
                kernel_ms[name] = round(kernel_ms.get(name, 0.0) + e.device_time_total / 1e3, 3)
        res["kernel_ms"] = kernel_ms
        g = kernel_ms.get("hap_gather_kernel")
        res["gather_GBps"] = round(2 * res["hap_bytes"] / (g * 1e-3) / 1e9, 1) if g else None
        eng.close()
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        res["gpu"] = q.stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
