"""Cost of --transcript_bam at config 2's batch size: one aligned transcriptome batch of N reads (default 262 144, dRNA model,
FASTQ) from T transcripts (default 40 000) spliced from spliced_bam_timing.py's seeded synthetic genome (4 x 25 Mb), in two
arms: without intron retention (the transcripts alone are resident) and with it (the genome resident behind them, the
batch's reads that retain an intron laid out on the genome as the CLI does: IntronRetention.plan_batch + ns_reemit, with
an IR Markov model of P(IR) 0.1 at the start and after a spliced intron, 0.5 after a retained one).  The GFF3, with exon
and intron features, is written by this tool and read back as the CLI reads it.  In each arm one context alternates
ns_compress_bam (unmapped records), ns_compress_bam_mapped (spliced records, ns_set_splice's map) and
ns_compress_bam_transcript (records against the transcripts) on the same batch.  Prints one JSON line, per arm:
  reads / chains   reads of the batch, and those that retain an intron
  calls_ms         host clock around each call, the three alternated on reused buffers (after one call each that grows them)
  kernels_ms       one more call each under torch.profiler with CUDA activities: device time by kernel name
  bytes            the members of each call
and gpu, the name and power limit read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import parity_checks as pc  # noqa: E402
from nanosim_b200 import _lib as L  # noqa: E402
from nanosim_b200.intron_retention import IntronRetention, TranscriptStructures, read_ir_markov_model  # noqa: E402
from nanosim_b200.records import name_table  # noqa: E402
from nanosim_b200.reference_fasta import PackedReference  # noqa: E402
from nanosim_b200.splice import build_splice_map  # noqa: E402
from spliced_bam_timing import synthetic  # noqa: E402


def add_introns(gff3):
    """Adds an intron feature between every two consecutive exons of a transcript (what intron retention reads)."""
    exons = {}
    lines = open(gff3).read().splitlines()
    for ln in lines[1:]:
        c = ln.split("\t")
        exons.setdefault(c[8], []).append((c[0], int(c[3]), int(c[4]), c[6]))
    for attr, ex in exons.items():
        ex.sort(key=lambda e: e[1])
        for (chrom, _, b, strand), (_, a, _, _) in zip(ex, ex[1:]):
            lines.append("%s\tsynthetic\tintron\t%d\t%d\t.\t%s\t.\t%s" % (chrom, b + 1, a - 1, strand, attr))
    with open(gff3, "w") as f:
        f.write("\n".join(lines) + "\n")


def kernels(f, names):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f(names)
    kern = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = ev.name.split("(")[0][:80]
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
    return {n: round(v, 3) for n, v in sorted(kern.items(), key=lambda kv: -kv[1])}


def run_arm(ir, trx, genome, st, d, args):
    n_trx = len(trx.names)
    w = np.random.default_rng(12).random(n_trx) + 0.1
    ref = PackedReference.concat(trx, genome) if ir else trx
    eng, _, _ = pc.make_trx_engine(ref, np.arange(n_trx, dtype=np.uint32), w / w.sum(), fastq=True, seed=13,
                                   trx_records=n_trx if ir else 0, max_len=trx.max_chrom)
    eng.set_splice(build_splice_map(st, trx.lengths, genome.lengths, n_trx if ir else None))
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, args.reads)
    res = {"reads": args.reads, "chains": 0}
    if ir:
        model = os.path.join(d, "IR_markov_model")
        with open(model, "w") as f:
            f.write("succedent\tno_IR\tIR\nstart\t0.9\t0.1\nno_IR\t0.9\t0.1\nIR\t0.5\t0.5\n")
        irm = IntronRetention(read_ir_markov_model(model), st, trx.lengths, n_trx)
        reads, pieces, ops = eng.fetch_meta()
        patch = irm.plan_batch(reads, pieces, ops, 0, 13, info.n_pieces, info.n_ops, info.raw_ev_off)
        eng.reemit(*patch)
        res["chains"] = len(patch[0])
        info = eng.info
    res["bases"], res["n_ops"] = int(info.total_bases), int(info.n_ops)
    names = name_table(eng.fetch(), ref.names, 0, transcriptome=True)
    arms = {"bam": eng.compress_bam, "spliced": eng.compress_bam_mapped, "transcript": eng.compress_bam_transcript}
    res["bytes"] = {k: f(names) for k, f in arms.items()}                  # grows the context's buffers
    calls = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f(names)
            calls[k].append(round(1e3 * (time.perf_counter() - t0), 2))
    res["calls_ms"] = calls
    res["kernels_ms"] = {k: kernels(f, names) for k, f in arms.items()}
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reads", type=int, default=262144)
    ap.add_argument("--transcripts", type=int, default=40000)
    ap.add_argument("--chrom_len", type=int, default=25_000_000)
    ap.add_argument("--chroms", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    with tempfile.TemporaryDirectory() as d:
        gff3 = os.path.join(d, "annotation.gff3")
        genome, trx = synthetic(args.transcripts, args.chrom_len, args.chroms, 11, gff3)
        add_introns(gff3)
        st = TranscriptStructures.from_gff3(gff3, trx.names, genome.raw_names)
        res = {"transcripts": len(trx.names), "genome_bases": int(genome.genome_len)}
        for ir in (False, True):
            res["ir" if ir else "no_ir"] = run_arm(ir, trx, genome, st, d, args)
    res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                text=True).stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
