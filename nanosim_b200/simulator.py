#!/usr/bin/env python
"""Drop-in driver for the simulation stage: ``simulator.py genome ...`` with the reference's command line
(/root/reference/src/simulator.py:2070-2531) and output files (``<out>_aligned_reads.{fasta,fastq}``,
``<out>_aligned_error_profile``, ``<out>_unaligned_reads.{fasta,fastq}``), the per-read work done by the CUDA
library through the C ABI.

read_profile() / simulation() keep the reference's names and argument meaning:
  read_profile  -> loads the FASTA and the model directory, compiles the model tables and uploads both to HBM once;
  simulation    -> the orchestrator (:1571-1672): instead of forking ``num_threads`` workers that each loop over reads
                   it launches batches on the GPU; with torchrun (WORLD_SIZE>1) every rank simulates its contiguous
                   shard of read ids and rank 0 concatenates the per-rank sub-files in rank order, exactly like the
                   reference concatenates its per-worker sub-files (:1626-1639).
"""
import argparse
import os
import struct
import sys
import zlib
from textwrap import dedent
from time import strftime

import numpy as np

from . import _lib as L
from .engine import Engine
from .model import DeviceTables, load_model
from .pipeline import BatchPipeline
from .records import name_table, write_error_profile, write_records
from .reference_fasta import (POLYA_SCALE, MetaReference, PackedReference, read_abundance, read_expression,
                              read_polya_list)
from .model import build_alias

VERSION = "3.2.2-b200"

# BGZF end-of-file marker: an empty member (SAM/BAM format specification §4.1.2), once at the end of every .gz file
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
ERR_HEADER = b"Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n"      # first line of the error profile (:1634)


def bgzf_member(text):
    """``text`` (at most 64 KiB) as one BGZF member, compressed on the host with zlib: the error profile's header line."""
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(text) + c.flush()
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", 18 + len(payload) + 8 - 1) + payload +
            struct.pack("<II", zlib.crc32(text), len(text)))


def bam_header():
    """The BAM header of ``--bam`` files as one BGZF member: magic, the @HD and @PG lines, no reference sequences.  It
    carries no command line, so the decompressed file depends only on the simulated reads."""
    text = b"@HD\tVN:1.6\tSO:unknown\n@PG\tID:NanoSim\tPN:NanoSim\tVN:" + VERSION.encode() + b"\n"
    return bgzf_member(b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", 0))


def _log(msg):
    sys.stdout.write(strftime("%Y-%m-%d %H:%M:%S") + ": " + msg + "\n")
    sys.stdout.flush()


class Profile:
    """What read_profile() leaves in module globals in the reference."""

    def __init__(self):
        self.ref = None
        self.tables = None
        self.engine = None
        self.number_aligned = 0
        self.number_unaligned = 0
        self.max_chrom = 0
        self.perfect = False


def _dist_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


def _dist_init():
    import torch.distributed as dist
    if not dist.is_initialized():
        dist.init_process_group("gloo")       # host-side plumbing only (objects, barriers); the reference travels over NCCL
    return dist


class _RemoteReference(PackedReference):
    """The reference as a rank other than 0 sees it before the broadcast: names and offsets, no bases yet."""

    def __init__(self, names, offsets, raw_names):
        self.names, self.raw_names = list(names), list(raw_names)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        self.bases = None


def read_profile(ref_g, number_list, model_prefix, per, mode, strandness, ref_t=None, dna_type=None, abun=None,
                 polya=None, exp=None, model_ir=False, chimeric=False, homopolymer=False, fastq=False,
                 device=0, seed=0, ir_files=None, ref_on_host=True):
    """read_profile (:244-591).  Under torchrun (WORLD_SIZE > 1) only rank 0 reads the reference files; the other ranks get
    names and offsets through torch.distributed and the bases through ONE NCCL broadcast into their HBM (ns_bcast_nccl).
    ref_on_host: those ranks also copy the bases back to the host, which only the plain error profile's formatter reads."""
    rank, world = _dist_world()
    if world > 1:
        return _read_profile_distributed(rank, world, ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun,
                                         polya, exp, model_ir, chimeric, homopolymer, fastq, device, seed, ir_files, ref_on_host)
    return _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp, model_ir,
                               chimeric, homopolymer, fastq, device, seed, ir_files)


def _read_profile_distributed(rank, world, ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp,
                              model_ir, chimeric, homopolymer, fastq, device, seed, ir_files, ref_on_host=True):
    dist = _dist_init()
    box = [None]
    if rank == 0:
        prof = _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp, model_ir,
                                   chimeric, homopolymer, fastq, device, seed, ir_files)
        r = prof.ref
        box[0] = {"names": r.names, "raw": r.raw_names, "offsets": r.offsets,
                  "meta": (r.species, r.chrom_species, r.chrom_circular, r.chrom_keys) if mode == "metagenome" else None,
                  "nccl_id": prof.engine.nccl_unique_id(),
                  "extra": {k: getattr(prof, k) for k in ("samples", "number_list", "expr_chrom", "expr_weights", "polya_flags", "max_chrom",
                                                          "n_trx", "coverage_ref_len", "counts", "number_aligned", "number_unaligned")
                            if hasattr(prof, k)}}
    dist.broadcast_object_list(box, src=0)
    info = box[0]
    if rank != 0:
        # everything of read_profile that is not the reference: model tables, counts, expression / abundance (from rank 0)
        prof = Profile()
        prof.ir, prof.n_trx = None, 0
        for k, v in info["extra"].items():
            setattr(prof, k, v)
        if info["meta"] is not None:
            sp, csp, circ, keys = info["meta"]
            prof.ref = MetaReference.__new__(MetaReference)
            _RemoteReference.__init__(prof.ref, info["names"], info["offsets"], info["raw"])
            prof.ref.species, prof.ref.chrom_species, prof.ref.chrom_circular, prof.ref.chrom_keys = sp, csp, circ, keys
        else:
            prof.ref = _RemoteReference(info["names"], info["offsets"], info["raw"])
        if mode == "transcriptome" and model_ir:
            from .intron_retention import IntronRetention, TranscriptStructures, read_ir_markov_model
            ir_files = ir_files or {}
            base = model_prefix[:-4] if model_prefix.endswith(".npz") else model_prefix
            n_trx = prof.n_trx
            trx_names, genome_raw = prof.ref.names[:n_trx], prof.ref.raw_names[n_trx:]
            st = TranscriptStructures.from_gff3(ir_files.get("gff3") or base + "_added_intron_final.gff3", trx_names, genome_raw)
            prof.ir = IntronRetention(read_ir_markov_model(ir_files.get("markov") or base + "_IR_markov_model"), st,
                                      prof.ref.lengths[:n_trx], n_trx)
        cm = load_model(model_prefix)
        prof.tables = DeviceTables(cm, fastq=fastq, homopolymer=homopolymer, chimeric=chimeric, perfect=per, strandness=strandness, mode=mode)
        prof.perfect, prof.seed = per, seed
        from .hostbind import bind_to_gpu_node
        bind_to_gpu_node(device)
        prof.engine = Engine(device=device, seed=seed)
    prof.engine.bcast_reference(info["nccl_id"], rank, world, 0)          # the one NCCL broadcast of the job
    if rank != 0:
        if ref_on_host:
            prof.ref.bases = prof.engine.reference_bases(int(prof.ref.offsets[-1]))   # host copy for the error profile's reference column
        prof.engine.ref = prof.ref
        prof.engine.set_model(prof.tables, perfect=per)
        if mode == "transcriptome":
            pr, al = build_alias(prof.expr_weights)
            prof.engine.set_expression(pr, al, prof.expr_chrom, prof.polya_flags)
    return prof


def _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t=None, dna_type=None, abun=None,
                        polya=None, exp=None, model_ir=False, chimeric=False, homopolymer=False, fastq=False,
                        device=0, seed=0, ir_files=None):
    prof = Profile()
    prof.ir = None
    prof.n_trx = 0
    _log("Read in reference ")
    if mode == "metagenome":
        try:
            prof.ref = MetaReference.from_genome_list(ref_g, dna_type)       # ref_g = genome list, dna_type = dna type list
            _log("Read in abundance profile")
            number_list, prof.samples = read_abundance(abun, prof.ref.species)
        except KeyError as e:
            sys.stderr.write(str(e).strip("'\"") + "\n")
            sys.exit(1)
        except ValueError as e:
            sys.stderr.write(str(e) + "\n")
            sys.exit(1)
        prof.number_list = number_list
    elif mode == "transcriptome":
        prof.ref = PackedReference.from_fasta(ref_t)
        prof.coverage_ref_len = prof.ref.genome_len      # -x counts the transcriptome only (:2348), not the IR genome
        _log("Read in expression profile")
        try:
            prof.expr_chrom, prof.expr_weights = read_expression(exp, prof.ref)
        except ValueError as e:
            sys.stderr.write(str(e) + "\n")
            sys.exit(1)
        prof.polya_flags = None
        if polya:
            _log("Read in list of transcripts with polyA tails")
            prof.polya_flags = read_polya_list(polya, prof.ref)
        prof.max_chrom = prof.ref.max_chrom
        if model_ir:
            # :404-453: the genome the retained introns are read from, the IR Markov model, the exon/intron structure
            from .intron_retention import IntronRetention, TranscriptStructures, read_ir_markov_model
            _log("Read in reference genome and create .fai index file")
            trx = prof.ref
            genome = PackedReference.from_fasta(ref_g)
            _log("Read in IR markov model")
            ir_files = ir_files or {}
            base = model_prefix[:-4] if model_prefix.endswith(".npz") else model_prefix
            p_no_ir = read_ir_markov_model(ir_files.get("markov") or base + "_IR_markov_model")
            _log("Read in GFF3 annotation file")
            st = TranscriptStructures.from_gff3(ir_files.get("gff3") or base + "_added_intron_final.gff3", trx.names, genome.raw_names)
            prof.n_trx = len(trx.names)
            prof.ir = IntronRetention(p_no_ir, st, trx.lengths, prof.n_trx)
            # :1094-1099: only transcripts whose GFF3 exons add up to their FASTA length are ever simulated
            from .intron_retention import expressed_with_structure
            prof.expr_chrom, prof.expr_weights, dropped = expressed_with_structure(prof.expr_chrom, prof.expr_weights, st, trx.lengths)
            if len(prof.expr_chrom) == 0:
                sys.stderr.write("No expressed transcript has a matching exon structure in the GFF3 annotation!\n")
                sys.exit(1)
            if dropped:
                _log("%d expressed transcripts without a matching exon structure are never drawn" % dropped)
            prof.ref = PackedReference.concat(trx, genome)
            if prof.polya_flags is not None:
                prof.polya_flags = np.concatenate([prof.polya_flags, np.zeros(len(genome.names), dtype=np.uint8)])
    else:
        prof.ref = PackedReference.from_fasta(ref_g)
    if mode != "transcriptome":
        prof.max_chrom = prof.ref.max_chrom
    if mode == "genome" and len(prof.ref.names) > 1 and dna_type == "circular":
        sys.stderr.write("Do not choose circular if there is more than one chromosome in the genome!\n")
        sys.exit(1)
    _log("Read error profile")
    cm = load_model(model_prefix)
    prof.tables = DeviceTables(cm, fastq=fastq, homopolymer=homopolymer, chimeric=chimeric, perfect=per,
                               strandness=strandness, mode=mode)
    prof.number_aligned, prof.number_unaligned = prof.tables.split_counts(number_list[0], per)
    prof.counts = [prof.tables.split_counts(n, per) for n in number_list]
    prof.perfect = per
    _log("Read KDF of aligned reads")
    prof.seed = seed
    # one process per GPU: keep its threads (record formatting, 2-bit expansion) and pinned buffers on the GPU's NUMA node
    from .hostbind import bind_to_gpu_node
    bind_to_gpu_node(device)
    prof.engine = Engine(device=device, seed=seed)
    prof.engine.set_reference(prof.ref)
    prof.engine.set_model(prof.tables, perfect=per)
    if mode == "transcriptome":
        pr, al = build_alias(prof.expr_weights)
        prof.engine.set_expression(pr, al, prof.expr_chrom, prof.polya_flags)
    return prof


def _shard(n, rank, world):
    per = n // world
    lo = rank * per
    hi = n if rank == world - 1 else lo + per        # remainder goes to the last worker (:1597-1598)
    return lo, hi


def simulation(prof, mode, out, dna_type, per, kmer_bias, basecaller, max_l, min_l, num_threads, fastq,
               median_l=None, sd_l=None, model_ir=False, uracil=False, polya=None, chimeric=False,
               batch_reads=65536, error_profile=True, rank=0, world=1, gzip=False, gzip_error_profile=False, bam=False):
    """gzip: write the reads as BGZF (``.gz``), compressed on the GPU; bam: write them as unaligned BAM (``.bam``, one
    unmapped record per read), encoded and compressed on the GPU.  The error profile stays plain text unless
    gzip_error_profile (needs gzip or bam): then it is formatted and compressed on the GPU too,
    ``<out>_aligned_error_profile.gz``, whose first member is the header line.  Under torchrun (world > 1) the per-rank
    files carry neither the headers nor the end-of-file block: merge_rank_files writes them."""
    fmt_threads = max(1, min(num_threads, os.cpu_count() or 1))     # host threads of the record formatter
    eng = prof.engine
    meta = mode == "metagenome"
    trx = mode == "transcriptome"
    lo_a, hi_a = _shard(prof.number_aligned, rank, world)
    eng.configure(circular=(dna_type == "circular"), perfect=per, fastq=fastq, chimeric=chimeric,
                  kmer_bias=kmer_bias or 0, min_len=min_l, max_len=max_l, median_len=median_l or 0.0, sd_len=sd_l or 0.0,
                  metagenome=meta, transcriptome=trx, uracil=bool(uracil),
                  polya_scale=POLYA_SCALE.get(basecaller, POLYA_SCALE["guppy"]) if (trx and polya) else 0.0,
                  # the reference's 2-D KDE sample has one row per read of a WORKER (:1072): -t sets its size as it does there
                  kde2d_sample=max(1, (hi_a - lo_a) // max(1, num_threads)),
                  trx_records=prof.n_trx if (trx and prof.ir is not None) else 0)
    ext = ".bam" if bam else (".fastq" if fastq else ".fasta") + (".gz" if gzip else "")
    suffix = "" if world == 1 else str(rank)
    want_err = error_profile and not per
    gz_err = (gzip or bam) and gzip_error_profile and want_err
    pipe = BatchPipeline(eng, depth=2, fetch=True, want_ops=want_err and not gz_err, compress_profile=gz_err, bam=bam)
    totals = {"reads": 0, "bases": 0, "bytes": 0}
    try:
        _simulation_body(prof, pipe, mode, out, per, fastq, meta, trx, ext, suffix, want_err, world, rank, batch_reads, fmt_threads, totals,
                         gzip, gz_err, bam)
    finally:
        pipe.close()         # the cloned contexts own device batch buffers and pinned staging
    return totals            # what this rank simulated and wrote (the reference returns nothing)


def _simulation_body(prof, pipe, mode, out, per, fastq, meta, trx, ext, suffix, want_err, world, rank, batch_reads, fmt_threads, totals,
                     gzip=False, gz_err=False, bam=False):
    packed = gzip or bam            # the records are compressed on the device: the batches arrive as BGZF members
    reads_header = bam_header() if bam and world == 1 else b""

    def jobs(kind, lo, hi):
        return [(kind, start, min(batch_reads, hi - start)) for start in range(lo, hi, batch_reads)]

    def put_members(f, data):
        view = memoryview(data)
        while len(view):
            w = os.pwrite(f.fd, view, f.pos)
            f.pos += w
            view = view[w:]

    def put_reads(f, b, names):
        if not packed:
            f.pos += write_records(f.fd, f.pos, b, names, fastq, n_threads=fmt_threads)
            return
        put_members(f, b.gz)

    def end_bgzf(f):
        if world == 1:
            f.pos += os.pwrite(f.fd, BGZF_EOF, f.pos)

    def end_reads(f):
        if packed:
            end_bgzf(f)

    class _Out:
        """An output file written at explicit offsets: the library's formatter threads pwrite() into it."""

        def __init__(self, path, header=b""):
            self.fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
            self.pos = 0
            if header:
                self.pos = os.pwrite(self.fd, header, 0)

        def close(self):
            os.close(self.fd)

    _log("Start simulation of aligned reads")
    lo, hi = _shard(prof.number_aligned, rank, world)
    f_reads = _Out(out + "_aligned_reads" + suffix + ext, reads_header)
    f_err = _Out(out + ("_aligned_error_profile" if world == 1 else "_error_profile" + suffix) + (".gz" if gz_err else ""),
                 b"" if world > 1 else bgzf_member(ERR_HEADER) if gz_err else ERR_HEADER)
    try:
        def aligned_names(b, job):
            return name_table(b, prof.ref.names, job[1], perfect=per, metagenome=meta, transcriptome=trx)

        def sink_aligned(info, b, job):
            names = b.names if packed else aligned_names(b, job)
            put_reads(f_reads, b, names)
            totals["reads"] += int(info.n_reads)
            totals["bases"] += int(info.total_bases)
            if gz_err:
                put_members(f_err, b.gz_err)
            elif want_err:
                f_err.pos += write_error_profile(f_err.fd, f_err.pos, b, names, prof.ref, seed=prof.seed, n_threads=fmt_threads)

        def retain_introns(engine, info, job):
            # intron retention (:1156-1183): decided on the host from the batch's metadata, the few affected reads are laid
            # out on the genome and emitted again (intron_retention.py)
            reads, pieces, ops = engine.fetch_meta()
            patch = prof.ir.plan_batch(reads, pieces, ops, job[1], prof.seed, info.n_pieces, info.n_ops, info.raw_ev_off)
            if patch is not None:
                engine.reemit(*patch)

        pipe.compress = aligned_names if packed else None
        pipe.run(jobs(L.NS_KIND_ALIGNED, lo, hi), sink_aligned, static_assign=meta,
                 after_simulate=retain_introns if (trx and prof.ir is not None and not per) else None)
        end_reads(f_reads)
        if gz_err:
            end_bgzf(f_err)
    finally:
        totals["bytes"] += f_reads.pos + f_err.pos
        f_reads.close()
        f_err.close()
    if not per:
        _log("Start simulation of random reads")
        lo, hi = _shard(prof.number_unaligned, rank, world)
        pipe.want_ops = pipe.compress_profile = False      # unaligned reads are not logged (:1482-1549)
        f_un = _Out(out + "_unaligned_reads" + suffix + ext, reads_header)
        try:
            def unaligned_names(b, job):
                # the reference's read index keeps counting after the aligned reads (shared total_simulated, :1574)
                return name_table(b, prof.ref.names, prof.number_aligned + job[1])

            def sink_unaligned(info, b, job):
                put_reads(f_un, b, b.names if packed else unaligned_names(b, job))
                totals["reads"] += int(info.n_reads)
                totals["bases"] += int(info.total_bases)

            pipe.compress = unaligned_names if packed else None
            pipe.run(jobs(L.NS_KIND_UNALIGNED, lo, hi), sink_unaligned, static_assign=meta)
            end_reads(f_un)
        finally:
            totals["bytes"] += f_un.pos
            f_un.close()


def merge_rank_files(out, fastq, per, world, gzip=False, gzip_error_profile=False, bam=False):
    """Rank 0: concatenate per-rank sub-files in rank order and delete them (:1626-1639, :1667-1672).  gzip: the reads
    files are BGZF members without an end-of-file block; the merged file gets it once, at its end.  bam: so are the
    ``.bam`` reads files, and the merged ones start with the BAM header's member.  gzip_error_profile: so are the
    error-profile files (``_error_profile{r}.gz``); the merged one starts with the header line's member."""
    ext = ".bam" if bam else (".fastq" if fastq else ".fasta") + (".gz" if gzip else "")
    header = bam_header() if bam else b""
    trailer = BGZF_EOF if gzip or bam else b""
    jobs = [("_aligned_reads%d" + ext, "_aligned_reads" + ext, header, trailer)]
    if gzip_error_profile:
        jobs.append(("_error_profile%d.gz", "_aligned_error_profile.gz", bgzf_member(ERR_HEADER), BGZF_EOF))
    else:
        jobs.append(("_error_profile%d", "_aligned_error_profile", ERR_HEADER, b""))
    if not per:
        jobs.append(("_unaligned_reads%d" + ext, "_unaligned_reads" + ext, header, trailer))
    for pat, dst, header, end in jobs:
        with open(out + dst, "wb") as o:
            o.write(header)
            for r in range(world):
                p = out + (pat % r)
                with open(p, "rb") as i:
                    while True:
                        blk = i.read(1 << 24)
                        if not blk:
                            break
                        o.write(blk)
                os.remove(p)
            o.write(end)


GZIP_HELP = ('Write the reads as BGZF-compressed <out>_aligned_reads.fast{a,q}.gz and <out>_unaligned_reads.fast{a,q}.gz, '
             'compressed on the GPU (gzip, zcat and samtools read them). The error profile stays plain text unless '
             '--gzip_error_profile is given (Default = False)')
GZIP_ERR_HELP = ('With --gzip or --bam: write the error profile as BGZF-compressed <out>_aligned_error_profile.gz, formatted and '
                 'compressed on the GPU (Default = False)')
BAM_HELP = ('Write the reads as unaligned BAM, <out>_aligned_reads.bam and <out>_unaligned_reads.bam (one unmapped record per '
            'read, as Dorado writes them), encoded and compressed on the GPU. The error profile stays plain text unless '
            '--gzip_error_profile is given (Default = False)')


def _plain_error_profile(args):
    """The run writes the error profile as plain text, formatted on the host from a host copy of the reference."""
    return not (args.no_error_profile or args.perfect or args.gzip_error_profile)


def build_parser():
    parser = argparse.ArgumentParser(
        description=dedent('''
        Simulation step
        -----------------------------------------------------------
        Given error profiles, reference genome, metagenome,
        and/or transcriptome, simulate ONT DNA or RNA reads
        '''), formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('-v', '--version', action='version', version='NanoSim ' + VERSION)
    sub = parser.add_subparsers(help="You may run the simulator on genome, transcriptome, or metagenome mode.", dest='mode')
    g = sub.add_parser('genome', help="Run the simulator on genome mode")
    g.add_argument('-rg', '--ref_g', help='Input reference genome', required=True)
    g.add_argument('-c', '--model_prefix', help='Location and prefix of error profiles generated from '
                   'characterization step (Default = training)', default="training")
    g.add_argument('-o', '--output', help='Output location and prefix for simulated reads (Default = simulated)',
                   default="simulated")
    g.add_argument('-n', '--number', help='Number of reads to be simulated (Default = 20000)', type=int, default=20000)
    g.add_argument('-x', '--coverage', help='Coverage of the simulated reads, overrides the number of reads', type=float,
                   default=None)
    g.add_argument('-max', '--max_len', help='The maximum length for simulated reads (Default = Infinity)', type=int,
                   default=float("inf"))
    g.add_argument('-min', '--min_len', help='The minimum length for simulated reads (Default = 50)', type=int, default=50)
    g.add_argument('-med', '--median_len', help='The median read length (Default = None)', type=int, default=None)
    g.add_argument('-sd', '--sd_len', help='The standard deviation of read length in log scale (Default = None)',
                   type=float, default=None)
    g.add_argument('--seed', help='Manually seeds the pseudo-random number generator', type=int, default=None)
    g.add_argument('-hp', '--homopolymer', help='Simulate homopolymer lengths (Default = False)', action='store_true',
                   default=False)
    g.add_argument('-k', '--KmerBias', help='Minimum homopolymer length to simulate homopolymer contraction and '
                   'expansion events in, a typical k is 5', type=int, default=None)
    g.add_argument('-s', '--strandness', help='Proportion of sense sequences. Overrides the value profiled in '
                   'characterization stage. Should be between 0 and 1', type=float, default=None)
    g.add_argument('-dna_type', help='Specify the dna type: circular OR linear (Default = linear)',
                   choices=["linear", "circular"], default="linear")
    g.add_argument('--perfect', help='Ignore error profiles and simulate perfect reads', action='store_true', default=False)
    g.add_argument('--fastq', help='Output fastq files instead of fasta files', action='store_true', default=False)
    g.add_argument('--chimeric', help='Simulate chimeric reads', action='store_true', default=False)
    g.add_argument('-t', '--num_threads', help='Number of host threads used for record formatting (Default = 1)',
                   type=int, default=1)
    # additions of this build
    g.add_argument('--batch_reads', help='Reads simulated per GPU batch (Default = 65536)', type=int, default=65536)
    g.add_argument('--no_error_profile', help='Skip writing <out>_aligned_error_profile', action='store_true', default=False)
    g.add_argument('--device', help='CUDA device index (Default = LOCAL_RANK or 0)', type=int, default=None)
    g.add_argument('--gzip', help=GZIP_HELP, action='store_true', default=False)
    g.add_argument('--gzip_error_profile', help=GZIP_ERR_HELP, action='store_true', default=False)
    g.add_argument('--bam', help=BAM_HELP, action='store_true', default=False)
    mg = sub.add_parser('metagenome', help="Run the simulator on metagenome mode")
    mg.add_argument('-gl', '--genome_list', help="Reference metagenome list, tsv file, the first column is species/strain "
                    "name, the second column is the reference genome fasta/fastq file directory", required=True)
    mg.add_argument('-a', '--abun', help="Abundance list, tsv file with header, the abundance of all species in each sample "
                    "need to sum up to 100", required=True)
    mg.add_argument('-dl', '--dna_type_list', help="DNA type list, tsv file, the first column is species/strain, the second "
                    "column is the chromosome name, the third column is the DNA type: circular OR linear")
    mg.add_argument('-c', '--model_prefix', help='Location and prefix of error profiles generated from characterization '
                    'step (Default = training)', default="training")
    mg.add_argument('-o', '--output', help='Output location and prefix for simulated reads (Default = simulated)',
                    default="simulated")
    mg.add_argument('-max', '--max_len', help='The maximum length for simulated reads (Default = Infinity)', type=int,
                    default=float("inf"))
    mg.add_argument('-min', '--min_len', help='The minimum length for simulated reads (Default = 50)', type=int, default=50)
    mg.add_argument('-med', '--median_len', help='The median read length (Default = None)', type=int, default=None)
    mg.add_argument('-sd', '--sd_len', help='The standard deviation of read length in log scale (Default = None)',
                    type=float, default=None)
    mg.add_argument('--seed', help='Manually seeds the pseudo-random number generator', type=int, default=None)
    mg.add_argument('-hp', '--homopolymer', help=argparse.SUPPRESS, action='store_true', default=False)
    mg.add_argument('-k', '--KmerBias', help=argparse.SUPPRESS, type=int, default=None)
    mg.add_argument('-s', '--strandness', help='Percentage of antisense sequences. Overrides the value profiled in '
                    'characterization stage. Should be between 0 and 1', type=float, default=None)
    mg.add_argument('--perfect', help='Ignore error profiles and simulate perfect reads', action='store_true', default=False)
    mg.add_argument('--abun_var', help='Simulate random variation in abundance values, takes in two values, format: '
                    'relative_var_low, relative_var_high, Example: -0.5 0.5)', nargs='+', type=float, default=None)
    mg.add_argument('--fastq', help='Output fastq files instead of fasta files', action='store_true', default=False)
    mg.add_argument('--chimeric', help='Simulate chimeric reads', action='store_true', default=False)
    mg.add_argument('-t', '--num_threads', help='Number of host threads used for record formatting (Default = 1)', type=int,
                    default=1)
    mg.add_argument('--batch_reads', help='Reads simulated per GPU batch (Default = 65536)', type=int, default=65536)
    mg.add_argument('--no_error_profile', help='Skip writing <out>_aligned_error_profile', action='store_true', default=False)
    mg.add_argument('--device', help='CUDA device index (Default = LOCAL_RANK or 0)', type=int, default=None)
    mg.add_argument('--gzip', help=GZIP_HELP, action='store_true', default=False)
    mg.add_argument('--gzip_error_profile', help=GZIP_ERR_HELP, action='store_true', default=False)
    mg.add_argument('--bam', help=BAM_HELP, action='store_true', default=False)
    t = sub.add_parser('transcriptome', help="Run the simulator on transcriptome mode")
    t.add_argument('-rt', '--ref_t', help='Input reference transcriptome', required=True)
    t.add_argument('-rg', '--ref_g', help='Input reference genome, required if intron retention simulation is on', default='')
    t.add_argument('-e', '--exp', help='Expression profile in the specified format as described in README', required=True)
    t.add_argument('-c', '--model_prefix', help='Location and prefix of error profiles generated from characterization '
                   'step (Default = training)', default="training")
    t.add_argument('-o', '--output', help='Output location and prefix for simulated reads (Default = simulated)',
                   default="simulated")
    t.add_argument('-n', '--number', help='Number of reads to be simulated (Default = 20000)', type=int, default=20000)
    t.add_argument('-x', '--coverage', help='Coverage of the simulated reads, overrides the number of reads', type=float,
                   default=None)
    t.add_argument('-max', '--max_len', help='The maximum length for simulated unaligned reads (Default = Infinity)',
                   type=int, default=float("inf"))
    t.add_argument('-min', '--min_len', help='The minimum length for simulated unaligned reads (Default = 50)', type=int,
                   default=50)
    t.add_argument('--seed', help='Manually seeds the pseudo-random number generator', type=int, default=None)
    t.add_argument('-hp', '--homopolymer', help='Simulate homopolymer lengths (Default = False)', action='store_true',
                   default=False)
    t.add_argument('-k', '--KmerBias', help='Minimum homopolymer length to simulate homopolymer contraction and expansion '
                   'events in, a typical k is 6', type=int, default=None)
    t.add_argument('-b', '--basecaller', help='Simulate polyA tails with respect to chosen basecaller: albacore or guppy',
                   choices=["albacore", "guppy"], default=None)
    t.add_argument('-s', '--strandness', help='Proportion of sense sequences. Overrides the value profiled in '
                   'characterization stage. Should be between 0 and 1', type=float, default=None)
    t.add_argument('--no_model_ir', help='Ignore simulating intron retention events', action='store_false', default=True)
    t.add_argument('--ir_markov_model', help='IR Markov model (Default = <model_prefix>_IR_markov_model)', default=None)
    t.add_argument('--ir_gff3', help='GFF3 with exon and intron features (Default = <model_prefix>_added_intron_final.gff3)',
                   default=None)
    t.add_argument('--perfect', help='Ignore profiles and simulate perfect reads', action='store_true', default=False)
    t.add_argument('--polya', help='Simulate polyA tails for given list of transcripts', default=None)
    t.add_argument('--fastq', help='Output fastq files instead of fasta files', action='store_true', default=False)
    t.add_argument('-t', '--num_threads', help='Number of host threads used for record formatting (Default = 1)', type=int,
                   default=1)
    t.add_argument('--uracil', help='Converts the thymine (T) bases to uracil (U) in the output fasta format',
                   action='store_true', default=False)
    t.add_argument('--batch_reads', help='Reads simulated per GPU batch (Default = 65536)', type=int, default=65536)
    t.add_argument('--no_error_profile', help='Skip writing <out>_aligned_error_profile', action='store_true', default=False)
    t.add_argument('--device', help='CUDA device index (Default = LOCAL_RANK or 0)', type=int, default=None)
    t.add_argument('--gzip', help=GZIP_HELP, action='store_true', default=False)
    t.add_argument('--gzip_error_profile', help=GZIP_ERR_HELP, action='store_true', default=False)
    t.add_argument('--bam', help=BAM_HELP, action='store_true', default=False)
    return parser, g, mg, t


def add_abundance_var(expected, total_len, var_low, var_high, rnd):
    """add_abundance_var (:594-615): largest |variation| to the species with the largest genome, renormalised to 100."""
    n = len(expected)
    var = sorted((rnd.uniform(var_low, var_high) for _ in range(n)), key=abs)
    by_size = sorted(range(n), key=lambda k: total_len[k])
    per_species = [0.0] * n
    for v, k in zip(var, by_size):
        per_species[k] = v
    with_var = [e + e * per_species[k] for k, e in enumerate(expected)]
    tot = sum(with_var)
    return [a * 100 / tot for a in with_var]


def main_transcriptome(args, parser_t):
    """main(), transcriptome branch (:2322-2414)."""
    max_len, min_len = args.max_len, args.min_len
    model_ir = args.no_model_ir
    if args.homopolymer and (args.KmerBias is None or args.KmerBias < 0):
        print("\nPlease input proper kmer bias value >= 0 to simulate homopolymer contraction and expansion events from\n")
        parser_t.print_help(sys.stderr)
        sys.exit(1)
    if args.strandness and (args.strandness < 0 or args.strandness > 1):
        print("\nPlease input proper strandness value between 0 and 1\n")
        parser_t.print_help(sys.stderr)
        sys.exit(1)
    if max_len < min_len:
        sys.stderr.write("\nMaximum read length must be longer than Minimum read length!\n")
        parser_t.print_help(sys.stderr)
        sys.exit(1)
    if model_ir and args.ref_g == '':
        sys.stderr.write("\nPlease provide a reference genome to simulate intron retention events!\n")
        parser_t.print_help(sys.stderr)
        sys.exit(1)
    if args.polya and args.basecaller is None:
        print("\nPlease input basecaller to simulate polyA tails from.\n")
        parser_t.print_help(sys.stderr)
        sys.exit(1)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.device if args.device is not None else int(os.environ.get("LOCAL_RANK", "0"))
    _log(' '.join(sys.argv))
    dir_name = os.path.dirname(args.output)
    if dir_name != '':
        os.makedirs(dir_name, exist_ok=True)
    number = [args.number]
    prof = read_profile(args.ref_g, number, args.model_prefix, args.perfect, "transcriptome", args.strandness,
                        ref_t=args.ref_t, dna_type="linear", model_ir=model_ir, polya=args.polya, exp=args.exp,
                        homopolymer=args.homopolymer, fastq=args.fastq, device=device, seed=args.seed or 0,
                        ir_files={"markov": args.ir_markov_model, "gff3": args.ir_gff3}, ref_on_host=_plain_error_profile(args))
    if args.coverage is not None:
        number[0] = coverage_to_reads(prof, prof.tables.cm, args.coverage)
        prof.number_aligned, prof.number_unaligned = prof.tables.split_counts(number[0], args.perfect)
    max_len = min(max_len, prof.max_chrom)
    simulation(prof, "transcriptome", args.output, "transcriptome", args.perfect, args.KmerBias if args.homopolymer else None,
               args.basecaller, max_len, min_len, max(args.num_threads, 1), args.fastq, None, None, model_ir, args.uracil,
               args.polya, batch_reads=args.batch_reads, error_profile=not args.no_error_profile, rank=rank, world=world,
               gzip=args.gzip, gzip_error_profile=args.gzip_error_profile, bam=args.bam)
    if world > 1:
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("gloo")
        dist.barrier()
        if rank == 0:
            merge_rank_files(args.output, args.fastq, args.perfect, world, gzip=args.gzip,
                             gzip_error_profile=args.gzip_error_profile, bam=args.bam)
        dist.barrier()
    _log("Finished!")


def main_metagenome(args, parser_mg):
    """main(), metagenome branch (:2416-2527)."""
    import random

    max_len, min_len = args.max_len, args.min_len
    if args.homopolymer and (args.KmerBias is None or args.KmerBias < 0):
        print("\nPlease input proper kmer bias value >= 0 to simulate homopolymer contraction and expansion events from\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    if args.strandness and (args.strandness < 0 or args.strandness > 1):
        print("\nPlease input proper strandness value between 0 and 1\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    if (args.median_len and not args.sd_len) or (args.sd_len and not args.median_len):
        sys.stderr.write("\nPlease provide both mean and standard deviation of read length!\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    if args.median_len and args.sd_len and args.chimeric:
        sys.stderr.write("\nLognormal distributed reads cannot be chimeric!\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    if max_len < min_len:
        sys.stderr.write("\nMaximum read length must be longer than Minimum read length!\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    if args.perfect and args.chimeric:
        print("\nPerfect reads cannot be chimeric\n")
        parser_mg.print_help(sys.stderr)
        sys.exit(1)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.device if args.device is not None else int(os.environ.get("LOCAL_RANK", "0"))
    _log(' '.join(sys.argv))
    dir_name = os.path.dirname(args.output)
    if dir_name != '':
        os.makedirs(dir_name, exist_ok=True)
    prof = read_profile(args.genome_list, [], args.model_prefix, args.perfect, "metagenome", args.strandness,
                        dna_type=args.dna_type_list, abun=args.abun, chimeric=args.chimeric, homopolymer=args.homopolymer,
                        fastq=args.fastq, device=device, seed=args.seed or 0, ref_on_host=_plain_error_profile(args))
    rnd = random.Random(args.seed)
    L_ = prof.ref.lengths
    total_len = [int(L_[prof.ref.chrom_species == i].sum()) for i in range(len(prof.ref.species))]
    max_len = min(max_len, max(prof.ref.max_chrom_per_species.values()))          # :2525
    for s_idx, expected in enumerate(prof.samples):
        abun = add_abundance_var(expected, total_len, float(args.abun_var[0]), float(args.abun_var[1]), rnd) \
            if args.abun_var else list(expected)
        beta = prof.tables.abun_inflation
        inflated = [1 - (1 - a) * beta for a in abun] if args.chimeric else None           # inflate_abun (:2018-2022)
        prof.engine.set_abundance(abun, inflated)
        _log("Simulating sample sample%d" % s_idx)
        prof.number_aligned, prof.number_unaligned = prof.counts[s_idx]
        simulation(prof, "metagenome", args.output + "_sample%d" % s_idx, "metagenome", args.perfect, None, None, max_len,
                   min_len, max(args.num_threads, 1), args.fastq, args.median_len, args.sd_len, chimeric=args.chimeric,
                   batch_reads=args.batch_reads, error_profile=not args.no_error_profile, rank=rank, world=world, gzip=args.gzip,
                   gzip_error_profile=args.gzip_error_profile, bam=args.bam)
        if world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                dist.init_process_group("gloo")
            dist.barrier()
            if rank == 0:
                merge_rank_files(args.output + "_sample%d" % s_idx, args.fastq, args.perfect, world, gzip=args.gzip,
                                 gzip_error_profile=args.gzip_error_profile, bam=args.bam)
            dist.barrier()
    _log("Finished!")


def coverage_to_reads(prof, cm, coverage):
    """calculate_read_number_from_coverage (:2024-2068).  The reference estimates the mean read length from 10M KDE
    samples; gaussian kernel noise has zero mean, so the estimate equals the weighted mean of the training samples."""
    rate = prof.tables.aligned_ratio
    w_al = rate / (rate + 1) if rate is not None else 1.0
    mean = w_al * cm.kde["aligned_reads"][0].mean()
    if "unaligned_length" in cm.kde:
        mean += (1 - w_al) * cm.kde["unaligned_length"][0].mean()
    ref_len = getattr(prof, "coverage_ref_len", None) or prof.ref.genome_len
    return int(ref_len / mean * coverage)


def main(argv=None):
    parser, parser_g, parser_mg, parser_t = build_parser()
    args = parser.parse_args(argv)
    if args.mode is None:
        parser.print_help(sys.stderr)
        sys.exit(1)
    usage = None
    if args.bam and args.gzip:
        usage = "--bam and --gzip both choose the format of the reads: give one of them"
    elif args.bam and getattr(args, "uracil", False):
        usage = "--bam cannot be combined with --uracil: BAM has no code for U"
    elif args.gzip_error_profile and not (args.gzip or args.bam):
        usage = "--gzip_error_profile needs --gzip or --bam"
    if usage:
        sys.stderr.write("\n" + usage + "!\n")
        {"genome": parser_g, "metagenome": parser_mg, "transcriptome": parser_t}[args.mode].print_help(sys.stderr)
        sys.exit(1)
    # no profile is written with --no_error_profile or --perfect: nothing to compress
    args.gzip_error_profile = args.gzip_error_profile and not args.no_error_profile and not args.perfect
    if args.mode == "metagenome":
        return main_metagenome(args, parser_mg)
    if args.mode == "transcriptome":
        return main_transcriptome(args, parser_t)
    number = [args.number]
    max_len, min_len = args.max_len, args.min_len
    if args.homopolymer and (args.KmerBias is None or args.KmerBias < 0):
        print("\nPlease input proper kmer bias value >= 0 to simulate homopolymer contraction and expansion events from\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)
    if args.strandness and (args.strandness < 0 or args.strandness > 1):
        print("\nPlease input proper strandness value between 0 and 1\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)
    if (args.median_len and not args.sd_len) or (args.sd_len and not args.median_len):
        sys.stderr.write("\nPlease provide both mean and standard deviation of read length!\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)
    if args.median_len and args.sd_len and args.chimeric:
        sys.stderr.write("\nLognormal distributed reads cannot be chimeric!\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)
    if max_len < min_len:
        sys.stderr.write("\nMaximum read length must be longer than Minimum read length!\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)
    if args.perfect and args.chimeric:
        print("\nPerfect reads cannot be chimeric\n")
        parser_g.print_help(sys.stderr)
        sys.exit(1)

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    device = args.device if args.device is not None else int(os.environ.get("LOCAL_RANK", "0"))
    _log(' '.join(sys.argv))
    dir_name = os.path.dirname(args.output)
    if dir_name != '':
        os.makedirs(dir_name, exist_ok=True)

    prof = read_profile(args.ref_g, number, args.model_prefix, args.perfect, args.mode, args.strandness,
                        dna_type=args.dna_type, chimeric=args.chimeric, homopolymer=args.homopolymer, fastq=args.fastq,
                        device=device, seed=args.seed or 0, ref_on_host=_plain_error_profile(args))
    if args.coverage is not None:
        number[0] = coverage_to_reads(prof, prof.tables.cm, args.coverage)
        prof.number_aligned, prof.number_unaligned = prof.tables.split_counts(number[0], args.perfect)
    max_len = min(max_len, prof.max_chrom)
    simulation(prof, args.mode, args.output, args.dna_type, args.perfect, args.KmerBias if args.homopolymer else None,
               None, max_len, min_len, max(args.num_threads, 1), args.fastq, args.median_len, args.sd_len,
               chimeric=args.chimeric, batch_reads=args.batch_reads, error_profile=not args.no_error_profile,
               rank=rank, world=world, gzip=args.gzip, gzip_error_profile=args.gzip_error_profile, bam=args.bam)
    if world > 1:
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("gloo")
        dist.barrier()
        if rank == 0:
            merge_rank_files(args.output, args.fastq, args.perfect, world, gzip=args.gzip,
                             gzip_error_profile=args.gzip_error_profile, bam=args.bam)
        dist.barrier()
    _log("Finished!")


if __name__ == "__main__":
    main()
