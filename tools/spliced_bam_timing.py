"""Cost of --spliced_bam at config 2's batch size: one aligned transcriptome batch of N reads (default 262 144, dRNA model,
FASTQ) on a seeded synthetic genome (4 x 25 Mb) with T transcripts (default 40 000, 2-12 exons of 80-600 bases, introns of
100-20 000 bases, strands alternating) spliced from it; their GFF3 is written by this tool and read back as the CLI reads
it.  The map is set with ns_set_splice; on the same batch the tool times ns_compress_bam (unmapped records) against
ns_compress_bam_mapped (spliced records).  Prints one JSON line:
  set_splice_ms    host clock around ns_set_splice (it ends in a device synchronise): checks, table, uploads
  splice_bytes     the device bytes the map keeps
  calls_ms         host clock around each call, arms alternated on reused buffers (after one call each that grows them)
  kernels_ms       per arm, one more call under torch.profiler with CUDA activities: device time by kernel name
  gpu              name and power limit, read in the same run."""
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

import parity_checks as pc  # noqa: E402
from nanosim_b200 import _lib as L  # noqa: E402
from nanosim_b200.intron_retention import TranscriptStructures  # noqa: E402
from nanosim_b200.records import name_table  # noqa: E402
from nanosim_b200.reference_fasta import PackedReference  # noqa: E402
from nanosim_b200.splice import build_splice_map  # noqa: E402

COMP = np.frombuffer(b"TGCA", dtype=np.uint8)


def synthetic(n_trx, chrom_len, n_chrom, seed, gff3):
    """(genome records, transcript records) of a seeded genome and transcripts spliced from it; writes their GFF3."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    codes = [rng.integers(0, 4, chrom_len).astype(np.uint8) for _ in range(n_chrom)]
    genome = [("chr%d" % (c + 1), acgt[codes[c]]) for c in range(n_chrom)]
    trx, lines = [], ["##gff-version 3"]
    per = n_trx // n_chrom
    for c in range(n_chrom):
        cursor = 1000
        for j in range(per):
            i = c * per + j
            minus = i % 2 == 1
            n_exon = int(rng.integers(2, 13))
            ex, pos = [], cursor + int(rng.integers(0, 2000))
            for e in range(n_exon):
                el = int(rng.integers(80, 601))
                ex.append((pos, pos + el))
                pos += el + int(rng.integers(100, 20001))
            if ex[-1][1] + 100 > chrom_len:
                cursor = 1000                                   # wrap: transcripts of a chromosome may overlap
                continue
            cursor = ex[0][1]
            tid = "ENST%011d" % i
            seq = np.concatenate([codes[c][a:b] for a, b in ex])
            seq = COMP[seq[::-1]] if minus else acgt[seq]
            trx.append((tid, seq))
            for a, b in ex:
                lines.append("chr%d\tsynthetic\texon\t%d\t%d\t.\t%s\t.\tParent=transcript:%s;transcript_id=%s"
                             % (c + 1, a + 1, b, "-" if minus else "+", tid, tid))
    with open(gff3, "w") as f:
        f.write("\n".join(lines) + "\n")
    return PackedReference.from_records(genome), PackedReference.from_records(trx)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reads", type=int, default=262144)
    ap.add_argument("--transcripts", type=int, default=40000)
    ap.add_argument("--chrom_len", type=int, default=25_000_000)
    ap.add_argument("--chroms", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    ap.add_argument("--tags", action="store_true", help="also time spliced records with NM and SA (ns_set_aln_tags), in a "
                    "second context that simulates the same batch")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        gff3 = os.path.join(d, "annotation.gff3")
        genome, trx = synthetic(args.transcripts, args.chrom_len, args.chroms, 11, gff3)
        st = TranscriptStructures.from_gff3(gff3, trx.names, genome.raw_names)
    smap = build_splice_map(st, trx.lengths, genome.lengths)
    res = {"reads": args.reads, "transcripts": len(trx.names), "exons": int(smap.exon_off[-1]), "genome_bases": int(genome.genome_len)}
    w = np.random.default_rng(12).random(len(trx.names)) + 0.1
    eng, _, _ = pc.make_trx_engine(trx, np.arange(len(trx.names), dtype=np.uint32), w / w.sum(), fastq=True, seed=13)
    t0 = time.perf_counter()
    res["splice_bytes"] = eng.set_splice(smap)
    res["set_splice_ms"] = round(1e3 * (time.perf_counter() - t0), 2)
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, args.reads)
    res["bases"], res["n_ops"] = int(info.total_bases), int(info.n_ops)
    names = name_table(eng.fetch(), trx.names, 0, transcriptome=True)
    arms = {"bam": eng.compress_bam, "spliced": eng.compress_bam_mapped}
    if args.tags:
        tagged, _, _ = pc.make_trx_engine(trx, np.arange(len(trx.names), dtype=np.uint32), w / w.sum(), fastq=True, seed=13)
        tagged.set_splice(smap)
        res["tags_bytes"] = tagged.set_aln_tags(list(genome.raw_names))
        tagged.simulate(L.NS_KIND_ALIGNED, 0, args.reads)
        arms["spliced_tagged"] = tagged.compress_bam_mapped
    res["bytes"] = {k: f(names) for k, f in arms.items()}                  # grows the context's buffers
    calls = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f(names)
            calls[k].append(round(1e3 * (time.perf_counter() - t0), 2))
    res["calls_ms"] = calls

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    res["kernels_ms"] = {}
    for k, f in arms.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f(names)
        kern = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name.split("(")[0][:80]
                kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
        res["kernels_ms"][k] = {n: round(v, 3) for n, v in sorted(kern.items(), key=lambda kv: -kv[1])}
    eng.close()
    if args.tags:
        tagged.close()
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                text=True).stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
