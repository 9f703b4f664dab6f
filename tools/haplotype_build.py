"""genome --vcf at config 2's scale: a 3.09 Gb synthetic genome (hg38 chromosome lengths, i.i.d. ACGT, as bench.py builds
it) and a synthetic VCF of about 4 M variants on it (SNVs, deletions and insertions of up to 10 and 20 bases, GT 0|1,
1|0 or 1|1); with --sv N, also about N structural variants (<DEL>, <INV>, <DUP>).  Prints one JSON line:
  parse_s          host time of variants.read_vcf (read, parse, check, tables)
  call_ms          the whole ns_apply_variants call between CUDA events (it ends in a device synchronise): host checks of
                   the tables, their upload, segments, scan, gather, and ns_set_reference on the haplotypes
  kernel_ms        device time of each of the build's kernels, from torch.profiler in a second build of its own
  hap_bytes, gather_GBps    bytes of the haplotypes, and 2 x that (read + write) over hap_gather_kernel's time
  accounted_peak_bytes      the sizes of the library's allocations at the build's peak (ns_apply_variants' count, not a
                   device reading)
  applied_sv, sv_bases       (--sv) the SV alleles applied per type, and the reference bases they cover
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


def sv_spans(ref, n_sv, seed=9):
    """About n_sv disjoint structural variants: <DEL>, <INV> and <DUP> equally, lengths log-uniform from 50 b to 1 Mb,
    plus a 10 Mb inversion on each of the first four chromosomes.  Per chromosome: (POS, END, type) arrays, sorted."""
    rng = np.random.default_rng(seed)
    L = ref.lengths
    out = []
    for c in range(len(L)):
        n = int(n_sv * L[c] / L.sum())
        size = np.exp(rng.uniform(np.log(50), np.log(1e6), n)).astype(np.int64)
        kind = rng.choice(3, n)
        if c < 4:
            size, kind = np.concatenate([size, [10_000_000]]), np.concatenate([kind, [1]])
        order = rng.permutation(len(size))
        size, kind = size[order], kind[order]
        while (size + 1).sum() + 1 > L[c]:
            size, kind = size[:-1], kind[:-1]
        free = int(L[c] - (size + 1).sum() - 1)
        gap = np.diff(np.concatenate([[0], np.sort(rng.integers(0, free + 1, len(size)))]))
        pos = 1 + np.cumsum(gap) + np.concatenate([[0], np.cumsum(size + 1)[:-1]])           # span [POS-1, END)
        out.append((pos, pos + size, kind))
    return out


def write_vcf(path, ref, n_variants, seed=7, svs=None):
    """svs (sv_spans): the structural variants too, and no small variant inside their spans on the same haplotype."""
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
        rows = []
        for p, r, k, s, i, g in zip(pos.tolist(), refs, kind.tolist(), snv.tolist(), ins, gts.tolist()):
            alt = (s if s != r[0] else "A" if r[0] != "A" else "C") if k == 0 else r[0] if k == 1 else r[0] + i
            rows.append((p, "%s\t%d\t.\t%s\t%s\t50\tPASS\t.\tGT\t%s\n" % (name, p, r, alt, g)))
        if svs is not None:
            sp, se, sk = svs[c]
            sgt = np.array(["0|1", "1|0", "1|1"])[rng.choice(3, len(sp), p=[0.4, 0.4, 0.2])]
            hap_mask = {"1|0": 1, "0|1": 2, "1|1": 3}
            j = np.searchsorted(sp - 1, pos - 1 + rlen) - 1              # the last SV span starting before the variant ends
            inside = (j >= 0) & (se[np.maximum(j, 0)] > pos - 1)
            shared = np.array([hap_mask[g] for g in gts.tolist()]) & np.array([hap_mask[g] for g in sgt.tolist()] + [0])[j]
            rows = [row for row, x in zip(rows, (inside & (shared > 0)).tolist()) if not x]     # the other haplotype is free
            for p, e, k, g in zip(sp.tolist(), se.tolist(), sk.tolist(), sgt.tolist()):
                info = "SVTYPE=DEL;SVLEN=%d" % (p - e) if k == 0 else "SVTYPE=%s;END=%d" % (("INV", "DUP")[k - 1], e)
                rows.append((p, "%s\t%d\t.\t%s\t<%s>\t50\tPASS\t%s\tGT\t%s\n" % (name, p, chr(ref.bases[base + p - 1]),
                                                                                 ("DEL", "INV", "DUP")[k], info, g)))
            rows.sort(key=lambda x: x[0])
        lines += [row for _, row in rows]
    with open(path, "w") as f:
        f.writelines(lines)
    return len(lines) - 1


_COMP = np.arange(256, dtype=np.uint8)
for _a, _b in ("AT", "CG", "RY", "KM", "BV", "DH"):
    for _x, _y in ((_a, _b), (_a.lower(), _b.lower())):
        _COMP[ord(_x)], _COMP[ord(_y)] = ord(_y), ord(_x)


def splice(tables, ref, h, limit=None):
    """Haplotype record h spliced on the host from the tables (each variant by its kind), its first `limit` bytes."""
    c = tables.hap_chrom[h]
    seq = ref.bases[int(ref.offsets[c]):int(ref.offsets[c + 1])]
    parts, prev, size = [], 0, 0
    for j in range(int(tables.var_off[h]), int(tables.var_off[h + 1])):
        if limit is not None and size > limit:
            break
        p, o, n = int(tables.var_pos[j]), int(tables.alt_off[j]), int(tables.alt_len[j])
        k = int(tables.alt_kind[j])
        alt = tables.alt[o:o + n] if k == 0 else seq[o:o + n] if k == 1 else _COMP[seq[o:o + n][::-1]]
        parts += [seq[prev:p], alt]
        size += p - prev + n
        prev = p + int(tables.var_ref_len[j])
    parts.append(seq[prev:] if limit is None else seq[prev:prev + limit])
    out = np.concatenate(parts)
    return out if limit is None else out[:limit]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--variants", type=int, default=4_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="chromosome lengths x scale (1.0 = 3.09 Gb)")
    ap.add_argument("--sv", type=int, default=0, help="also about this many structural variants (<DEL>, <INV>, <DUP>; 50 b to "
                    "1 Mb, plus four 10 Mb inversions); small variants inside them on the same haplotype are left out")
    ap.add_argument("--parse-only", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()
    ref = genome(args.scale)
    res = {"genome_bases": ref.genome_len}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.vcf")
        res["vcf_records"] = write_vcf(path, ref, args.variants, svs=sv_spans(ref, args.sv) if args.sv else None)
        res["vcf_bytes"] = os.path.getsize(path)
        t0 = time.perf_counter()
        tables = read_vcf(path, ref)
        res["parse_s"] = round(time.perf_counter() - t0, 3)
    res["applied"] = int(tables.applied.sum())
    if args.sv:
        res["applied_sv"] = dict(zip(("del", "inv", "dup"), tables.structural.sum(axis=0).tolist()))
        res["sv_bases"] = int(tables.alt_len[tables.alt_kind > 0].sum() + tables.var_ref_len[(tables.alt_kind == 0) & (tables.alt_len == 0)].sum())
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
        # spot check against the tables spliced on the host: the first 1 MB of every haplotype record, and the whole of
        # the first chromosome's (which carries a 10 Mb inversion in the SV arm) and of the last record
        got = eng.reference_bases(res["hap_bytes"])
        offs = tables.offsets.astype(np.int64)
        n_hap = len(tables.hap_chrom)
        for h in range(n_hap):
            whole = tables.hap_chrom[h] == 0 or h == n_hap - 1
            want = splice(tables, ref, h, None if whole else 1 << 20)
            assert (not whole or len(want) == offs[h + 1] - offs[h]) and np.array_equal(got[offs[h]:offs[h] + len(want)], want), tables.names[h]
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
            key = e.key[len("void "):] if e.key.startswith("void ") else e.key        # templates: void name<args>(...)
            if key.startswith(("hap_", "pack_reference_kernel")) or "DeviceScan" in key:
                name = key.split("(")[0].split("<")[0] if key.startswith(("hap_", "pack_")) else "cub_scan"
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
