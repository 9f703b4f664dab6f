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
from collections import namedtuple
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
BGZF_HEADER_BLOCK = 56 << 10     # header bytes per member: zlib's output for them stays below the 64 KiB BGZF allows
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
ERR_HEADER = b"Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n"      # first line of the error profile (:1634)


def bgzf_member(text):
    """``text`` (at most 64 KiB) as one BGZF member, compressed on the host with zlib: the error profile's header line."""
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(text) + c.flush()
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", 18 + len(payload) + 8 - 1) + payload +
            struct.pack("<II", zlib.crc32(text), len(text)))


def bam_header(refs=None):
    """The BAM header of ``--bam`` files: magic, the @HD and @PG lines, no reference sequences, as one BGZF member.  It
    carries no command line, so the decompressed file depends only on the simulated reads.  refs (``--mapped_bam``): the
    reference records as (name, length, circular), which get one @SQ line each (``TP:circular`` on circular ones) and the
    binary reference list; that header is cut into members of at most BGZF_HEADER_BLOCK bytes."""
    refs = refs or []
    sq = b"".join(b"@SQ\tSN:%s\tLN:%d%s\n" % (n.encode(), ln, b"\tTP:circular" if c else b"") for n, ln, c in refs)
    text = b"@HD\tVN:1.6\tSO:unknown\n" + sq + b"@PG\tID:NanoSim\tPN:NanoSim\tVN:" + VERSION.encode() + b"\n"
    raw = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    raw += b"".join(struct.pack("<i", len(n.encode()) + 1) + n.encode() + b"\0" + struct.pack("<i", ln) for n, ln, _ in refs)
    return b"".join(bgzf_member(raw[k:k + BGZF_HEADER_BLOCK]) for k in range(0, len(raw), BGZF_HEADER_BLOCK))


def bam_refs(ref, circular=False):
    """The reference records of a mapped BAM header, as bam_header takes them: name (the FASTA header up to the first blank,
    or a --vcf haplotype's name), length and whether the record is circular (``-dna_type circular``, or the metagenome's
    DNA type list).  A name given to two records, and a record longer than BAM's int32 l_ref holds, are ValueErrors that
    name the record."""
    names, lengths = list(ref.raw_names), [int(x) for x in ref.lengths]
    for i, ln in enumerate(lengths):
        if ln > 0x7fffffff:
            raise ValueError("reference record %d (%s) has %d bases, more than the %d a BAM header can state"
                             % (i, ref.names[i], ln, 0x7fffffff))
    circ = getattr(ref, "chrom_circular", None)
    circ = [bool(c) for c in circ] if circ is not None else [bool(circular)] * len(names)
    seen = {}
    for i, n in enumerate(names):
        if n in seen:
            j = seen[n]
            raise ValueError("reference records %d (%s) and %d (%s) have the same name %s: a mapped BAM cannot tell them apart"
                             % (j, ref.names[j], i, ref.names[i], n))
        seen[n] = i
    return list(zip(names, lengths, circ))


# One output file of a run: <out><name>, or <out><rank_name % r> for rank r's part under torchrun, which has neither header
# nor trailer; members: its content arrives as BGZF members
OutputFile = namedtuple("OutputFile", "name rank_name header trailer members")


def output_files(fastq, gzip=False, gzip_error_profile=False, bam=False, mapped_refs=None):
    """What the format flags make of each output file: {"aligned", "error_profile", "unaligned"} -> OutputFile.  gzip and
    bam: the reads files are BGZF members that end with the end-of-file block, and bam's start with the BAM header (with
    mapped_refs' @SQ lines for the aligned reads).  gzip_error_profile: the error profile is BGZF members too, the first one
    its header line."""
    ext = ".bam" if bam else (".fastq" if fastq else ".fasta") + (".gz" if gzip else "")
    packed = gzip or bam
    trailer = BGZF_EOF if packed else b""
    header = bam_header() if bam else b""
    aligned_header = bam_header(mapped_refs) if bam and mapped_refs is not None else header
    err = ".gz" if gzip_error_profile else ""
    err_header = bgzf_member(ERR_HEADER) if gzip_error_profile else ERR_HEADER
    return {"aligned": OutputFile("_aligned_reads" + ext, "_aligned_reads%d" + ext, aligned_header, trailer, packed),
            "error_profile": OutputFile("_aligned_error_profile" + err, "_error_profile%d" + err, err_header,
                                        BGZF_EOF if gzip_error_profile else b"", gzip_error_profile),
            "unaligned": OutputFile("_unaligned_reads" + ext, "_unaligned_reads%d" + ext, header, trailer, packed)}


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
        self.haplotypes = None      # genome --vcf: variants.HaplotypeTables
        self.haploid = None         # genome --vcf: names and offsets of the haploid reference records


def _dist_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))


def _dist_init():
    import torch.distributed as dist
    if not dist.is_initialized():
        dist.init_process_group("gloo")       # host-side plumbing only (objects, barriers); the reference travels over NCCL
    return dist


class _RemoteReference(PackedReference):
    """A reference whose bases are in HBM only: names and offsets.  What a rank other than 0 sees before the broadcast,
    and the haplotype records of ``--vcf``, which are built on the device."""

    def __init__(self, names, offsets, raw_names):
        self.names, self.raw_names = list(names), list(raw_names)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        self.bases = None


def read_profile(ref_g, number_list, model_prefix, per, mode, strandness, ref_t=None, dna_type=None, abun=None,
                 polya=None, exp=None, model_ir=False, chimeric=False, homopolymer=False, fastq=False,
                 device=0, seed=0, ir_files=None, ref_on_host=True, vcf=None, lift=False, spliced=False, transcript=False):
    """read_profile (:244-591).  Under torchrun (WORLD_SIZE > 1) only rank 0 reads the reference files; the other ranks get
    names and offsets through torch.distributed and the bases through ONE NCCL broadcast into their HBM (ns_bcast_nccl).
    ref_on_host: those ranks also copy the bases back to the host, which only the plain error profile's formatter reads.
    vcf (genome mode): the reads come from the haplotypes of the VCF's first sample.  Rank 0 parses it and hands the
    tables to the other ranks; every rank builds the haplotypes in its HBM from the haploid reference (ns_apply_variants),
    and with ref_on_host copies them back to the host.  lift (``--lift_mapped_bam``): every rank also keeps the lift of the
    haplotypes onto the haploid records (ns_set_lift), so that mapped BAM records are against those.  spliced
    (transcriptome ``--spliced_bam``): rank 0 also builds the transcripts' map onto the genome records (prof.splice) and
    their header list (prof.spliced_refs) and hands both to the other ranks.  transcript (transcriptome ``--transcript_bam``)
    with intron retention: rank 0 builds the same map (prof.splice), which places the reads that retain an intron on their
    transcripts."""
    rank, world = _dist_world()
    if world > 1:
        return _read_profile_distributed(rank, world, ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun,
                                         polya, exp, model_ir, chimeric, homopolymer, fastq, device, seed, ir_files, ref_on_host, vcf,
                                         lift, spliced, transcript)
    prof = _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp, model_ir,
                               chimeric, homopolymer, fastq, device, seed, ir_files, vcf, spliced, transcript)
    if prof.haplotypes is not None:
        _apply_variants(prof, prof.haplotypes, ref_on_host, lift)
    return prof


def _apply_variants(prof, tables, ref_on_host, lift=False):
    """Makes the haplotype records of ``tables`` the resident reference of prof.engine (built on the device); the haploid
    records' names and offsets stay in prof.haploid.  lift: ns_set_lift with the same tables."""
    prof.haploid = _RemoteReference(prof.ref.names, prof.ref.offsets, prof.ref.raw_names)
    prof.haplotypes = tables
    prof.engine.apply_variants(tables)
    if lift:
        prof.engine.set_lift(tables)
    prof.ref = _RemoteReference(tables.names, tables.offsets, tables.names)
    if ref_on_host:
        prof.ref.bases = prof.engine.reference_bases(prof.ref.genome_len)
    prof.engine.ref = prof.ref
    for name, n, (n_del, n_inv, n_dup), skipped in zip(tables.names, tables.applied, tables.structural, tables.skipped):
        _log("%s: %d variants applied (of them from symbolic alleles: %d deletions, %d inversions, %d duplications), %d records of "
             "its chromosome skipped by FILTER" % (name, n, n_del, n_inv, n_dup, skipped))
    if tables.skipped_elsewhere:
        _log("%d records on contigs that are not in the reference skipped by FILTER" % tables.skipped_elsewhere)


def _read_profile_distributed(rank, world, ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp,
                              model_ir, chimeric, homopolymer, fastq, device, seed, ir_files, ref_on_host=True, vcf=None, lift=False,
                              spliced=False, transcript=False):
    dist = _dist_init()
    box = [None]
    if rank == 0:
        prof = _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t, dna_type, abun, polya, exp, model_ir,
                                   chimeric, homopolymer, fastq, device, seed, ir_files, vcf, spliced, transcript)
        r = prof.ref
        box[0] = {"names": r.names, "raw": r.raw_names, "offsets": r.offsets, "haplotypes": prof.haplotypes,
                  "meta": (r.species, r.chrom_species, r.chrom_circular, r.chrom_keys) if mode == "metagenome" else None,
                  "nccl_id": prof.engine.nccl_unique_id(),
                  "extra": {k: getattr(prof, k) for k in ("samples", "number_list", "expr_chrom", "expr_weights", "polya_flags", "max_chrom",
                                                          "n_trx", "coverage_ref_len", "counts", "number_aligned", "number_unaligned",
                                                          "splice", "spliced_refs")
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
    if info["haplotypes"] is not None:
        _apply_variants(prof, info["haplotypes"], ref_on_host, lift)
    if rank != 0:
        if ref_on_host and info["haplotypes"] is None:
            prof.ref.bases = prof.engine.reference_bases(int(prof.ref.offsets[-1]))   # host copy for the error profile's reference column
        prof.engine.ref = prof.ref
        prof.engine.set_model(prof.tables, perfect=per)
        if mode == "transcriptome":
            pr, al = build_alias(prof.expr_weights)
            prof.engine.set_expression(pr, al, prof.expr_chrom, prof.polya_flags)
    return prof


def _read_profile_local(ref_g, number_list, model_prefix, per, mode, strandness, ref_t=None, dna_type=None, abun=None,
                        polya=None, exp=None, model_ir=False, chimeric=False, homopolymer=False, fastq=False,
                        device=0, seed=0, ir_files=None, vcf=None, spliced=False, transcript=False):
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
        if spliced:
            _splice_profile(prof, ref_g, _gff3_path(model_prefix, ir_files), st if model_ir else None, genome if model_ir else None)
        elif transcript and model_ir:
            _splice_map(prof, st, genome, _gff3_path(model_prefix, ir_files), "those of their reads that retain an intron are written unmapped")
    else:
        prof.ref = PackedReference.from_fasta(ref_g)
    if mode != "transcriptome":
        prof.max_chrom = prof.ref.max_chrom
    if vcf:
        from .variants import VcfError, read_vcf
        _log("Read in VCF")
        try:
            prof.haplotypes = read_vcf(vcf, prof.ref)
        except VcfError as e:
            sys.stderr.write("%s: %s\n" % (vcf, e))
            sys.exit(1)
        prof.max_chrom = int(prof.haplotypes.lengths.max())
        prof.coverage_ref_len = prof.ref.genome_len         # -x counts the haploid reference
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


def _gff3_path(model_prefix, ir_files):
    """The GFF3 with the exon / intron features: --ir_gff3, else <model_prefix>_added_intron_final.gff3."""
    base = model_prefix[:-4] if model_prefix.endswith(".npz") else model_prefix
    return (ir_files or {}).get("gff3") or base + "_added_intron_final.gff3"


def _splice_profile(prof, ref_g, gff3, st=None, genome=None):
    """--spliced_bam: the map of the transcript records (the first ones of prof.ref) onto the -rg genome records
    (prof.splice) and the genome's header list (prof.spliced_refs).  With intron retention the genome and the structures
    are those it read, and the genome is resident behind the transcripts; without it only the genome's record names and
    lengths are kept (its bases never reach the device) and the GFF3 is read here."""
    from .intron_retention import TranscriptStructures
    n_trx = prof.n_trx or len(prof.ref.names)
    if genome is None:
        g = PackedReference.from_fasta(ref_g)
        genome = _RemoteReference(g.names, g.offsets, g.raw_names)
    try:
        prof.spliced_refs = bam_refs(genome)
    except ValueError as e:
        sys.stderr.write("\n--spliced_bam: %s!\n" % e)
        sys.exit(1)
    if st is None:
        _log("Read in GFF3 annotation file")
        st = TranscriptStructures.from_gff3(gff3, prof.ref.names[:n_trx], genome.raw_names)
    _splice_map(prof, st, genome, gff3, "their reads are written unmapped")


def _splice_map(prof, st, genome, gff3, unmapped):
    """The map of the transcript records (the first ones of prof.ref) onto the genome records by the structures st
    (prof.splice); the start-up log counts the expressed transcripts without one and says which of their reads
    (``unmapped``) that leaves unmapped."""
    from .splice import build_splice_map
    n_trx = prof.n_trx or len(prof.ref.names)
    prof.splice = build_splice_map(st, prof.ref.lengths[:n_trx], genome.lengths, n_trx if prof.n_trx else None)
    expressed = np.unique(np.asarray(prof.expr_chrom, dtype=np.int64))
    _log("%d expressed transcripts have no usable exon structure in %s: %s" % (int((~prof.splice.has_map()[expressed]).sum()), gff3, unmapped))


def _shard(n, rank, world):
    per = n // world
    lo = rank * per
    hi = n if rank == world - 1 else lo + per        # remainder goes to the last worker (:1597-1598)
    return lo, hi


def simulation(prof, mode, out, dna_type, per, kmer_bias, basecaller, max_l, min_l, num_threads, fastq,
               median_l=None, sd_l=None, model_ir=False, uracil=False, polya=None, chimeric=False,
               batch_reads=65536, error_profile=True, rank=0, world=1, gzip=False, gzip_error_profile=False, bam=False,
               mapped_refs=None, transcript_bam=False):
    """gzip: write the reads as BGZF (``.gz``), compressed on the GPU; bam: write them as unaligned BAM (``.bam``, one
    unmapped record per read), encoded and compressed on the GPU.  mapped_refs (with bam; bam_refs' list): the aligned
    reads are written as mapped records, their true alignments to those records (``--mapped_bam``); transcript_bam
    (transcriptome ``--transcript_bam``): to the transcript records, mapped_refs listing those.  The error profile stays plain text unless
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
    want_err = error_profile and not per
    gz_err = (gzip or bam) and gzip_error_profile and want_err
    files = output_files(fastq, gzip, gz_err, bam, mapped_refs)
    pipe = BatchPipeline(eng, depth=2, fetch=True, want_ops=want_err and not gz_err, compress_profile=gz_err, bam=bam,
                         mapped_bam=mapped_refs is not None, transcript_bam=transcript_bam)
    totals = {"reads": 0, "bases": 0, "bytes": 0}
    try:
        _simulation_body(prof, pipe, out, per, fastq, meta, trx, files, want_err, world, rank, batch_reads, fmt_threads, totals)
    finally:
        pipe.close()         # the cloned contexts own device batch buffers and pinned staging
    return totals            # what this rank simulated and wrote (the reference returns nothing)


def _simulation_body(prof, pipe, out, per, fastq, meta, trx, files, want_err, world, rank, batch_reads, fmt_threads, totals):
    packed = files["aligned"].members       # the records are compressed on the device: the batches arrive as BGZF members

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

    class _Out:
        """An output file written at explicit offsets: the library's formatter threads pwrite() into it."""

        def __init__(self, f):
            self.fd = os.open(out + (f.name if world == 1 else f.rank_name % rank), os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
            self.pos = os.pwrite(self.fd, f.header, 0) if world == 1 else 0
            self.trailer = f.trailer if world == 1 else b""        # under torchrun merge_rank_files writes both

        def end(self):
            self.pos += os.pwrite(self.fd, self.trailer, self.pos)

        def close(self):
            os.close(self.fd)

    _log("Start simulation of aligned reads")
    lo, hi = _shard(prof.number_aligned, rank, world)
    f_reads = _Out(files["aligned"])
    f_err = _Out(files["error_profile"])
    try:
        def aligned_names(b, job):
            return name_table(b, prof.ref.names, job[1], perfect=per, metagenome=meta, transcriptome=trx)

        def sink_aligned(info, b, job):
            names = b.names if packed else aligned_names(b, job)
            put_reads(f_reads, b, names)
            totals["reads"] += int(info.n_reads)
            totals["bases"] += int(info.total_bases)
            if files["error_profile"].members:
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
        f_reads.end()
        f_err.end()
    finally:
        totals["bytes"] += f_reads.pos + f_err.pos
        f_reads.close()
        f_err.close()
    if not per:
        _log("Start simulation of random reads")
        lo, hi = _shard(prof.number_unaligned, rank, world)
        pipe.want_ops = pipe.compress_profile = False      # unaligned reads are not logged (:1482-1549)
        f_un = _Out(files["unaligned"])
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
            f_un.end()
        finally:
            totals["bytes"] += f_un.pos
            f_un.close()


def merge_rank_files(out, fastq, per, world, gzip=False, gzip_error_profile=False, bam=False, mapped_refs=None):
    """Rank 0: concatenate per-rank sub-files in rank order and delete them (:1626-1639, :1667-1672), between each file's
    header and trailer (output_files)."""
    for key, f in output_files(fastq, gzip, gzip_error_profile, bam, mapped_refs).items():
        if key == "unaligned" and per:
            continue
        with open(out + f.name, "wb") as o:
            o.write(f.header)
            for r in range(world):
                p = out + (f.rank_name % r)
                with open(p, "rb") as i:
                    while True:
                        blk = i.read(1 << 24)
                        if not blk:
                            break
                        o.write(blk)
                os.remove(p)
            o.write(f.trailer)


GZIP_HELP = ('Write the reads as BGZF-compressed <out>_aligned_reads.fast{a,q}.gz and <out>_unaligned_reads.fast{a,q}.gz, '
             'compressed on the GPU (gzip, zcat and samtools read them). The error profile stays plain text unless '
             '--gzip_error_profile is given (Default = False)')
GZIP_ERR_HELP = ('With --gzip or --bam: write the error profile as BGZF-compressed <out>_aligned_error_profile.gz, formatted and '
                 'compressed on the GPU (Default = False)')
BAM_HELP = ('Write the reads as unaligned BAM, <out>_aligned_reads.bam and <out>_unaligned_reads.bam (one unmapped record per '
            'read, as Dorado writes them), encoded and compressed on the GPU. The error profile stays plain text unless '
            '--gzip_error_profile is given (Default = False)')
SPLICED_BAM_HELP = ('With --bam and -rg: write <out>_aligned_reads.bam as mapped records, the true spliced alignment of every '
                    'aligned read to the -rg genome records (N for every intron the read skips, XS:A for the transcript\'s strand), '
                    'built on the GPU with the exons of the GFF3 (--ir_gff3 or its default, also without intron retention). '
                    'Read names, the error profile and <out>_unaligned_reads.bam are unchanged (Default = False)')
MAPPED_BAM_HELP = ('With --bam: write <out>_aligned_reads.bam as mapped records, the true alignment of every aligned read to the '
                   'reference records (one record per segment, supplementary ones for chimeric reads, CIGAR from the simulated '
                   'errors), built on the GPU. <out>_unaligned_reads.bam is unchanged (Default = False)')
VCF_HELP = ('Simulate the reads from the haplotypes of the first sample of this VCF (plain or .vcf.gz), built on the GPU from '
            'the reference: records <chrom>-hap1 and <chrom>-hap2 (one copy for a haploid GT). Only FILTER PASS or . records '
            'are applied. -x still counts the haploid reference, so -x 30 is about 15x per haplotype')
LIFT_HELP = ('With --vcf and --mapped_bam: write the true alignments in <out>_aligned_reads.bam against the -rg records (as '
             'an aligner or a VCF names them) instead of the haplotype records: variants become CIGAR operations, <INV> and '
             '<DUP> split alignments, and every record has HP:C:1 or HP:C:2 for its haplotype. Read names and the error '
             'profile stay in haplotype coordinates (Default = False)')
TRANSCRIPT_BAM_HELP = ('With --bam: write <out>_aligned_reads.bam as mapped records, the true alignment of every aligned read '
                       'to the -rt transcript it was simulated from, built on the GPU. Bases of a retained intron are '
                       'insertions; with intron retention (the default) the exons of the GFF3 place those reads on the '
                       'transcript. Cannot be combined with --spliced_bam. Read names, the error profile and '
                       '<out>_unaligned_reads.bam are unchanged (Default = False)')
ALN_TAGS_HELP = ('With --mapped_bam (genome, metagenome; lifted or not) or --spliced_bam / --transcript_bam (transcriptome): '
                 'give every mapped record of <out>_aligned_reads.bam NM:I (edit distance to the reference bases, as samtools calmd counts it) '
                 'and, for a read with more than one record, SA:Z listing its other records, computed on the GPU. '
                 'Nothing else in the output changes (Default = False)')


def _set_aln_tags(args, prof, mapped_refs):
    """--aln_tags: NM and SA against the records of the mapped header (mapped_refs), with the REF bytes of the VCF's
    ALTs under --lift_mapped_bam; before simulation() clones the engine."""
    if not getattr(args, "aln_tags", False):
        return
    names = [n for n, _, _ in mapped_refs]
    if getattr(args, "lift_mapped_bam", False):
        t = prof.haplotypes
        prof.engine.set_aln_tags(names, t.ref_paired, len(t.var_pos))
    else:
        prof.engine.set_aln_tags(names)


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
    g.add_argument('--mapped_bam', help=MAPPED_BAM_HELP, action='store_true', default=False)
    g.add_argument('--vcf', help=VCF_HELP, default=None)
    g.add_argument('--lift_mapped_bam', help=LIFT_HELP, action='store_true', default=False)
    g.add_argument('--aln_tags', help=ALN_TAGS_HELP, action='store_true', default=False)
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
    mg.add_argument('--mapped_bam', help=MAPPED_BAM_HELP, action='store_true', default=False)
    mg.add_argument('--aln_tags', help=ALN_TAGS_HELP, action='store_true', default=False)
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
    t.add_argument('--mapped_bam', help=argparse.SUPPRESS, action='store_true', default=False)     # a usage error here
    t.add_argument('--spliced_bam', help=SPLICED_BAM_HELP, action='store_true', default=False)
    t.add_argument('--transcript_bam', help=TRANSCRIPT_BAM_HELP, action='store_true', default=False)
    t.add_argument('--aln_tags', help=ALN_TAGS_HELP, action='store_true', default=False)
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
    gff3 = _gff3_path(args.model_prefix, {"gff3": args.ir_gff3})
    if (args.spliced_bam or (args.transcript_bam and model_ir)) and not os.path.exists(gff3):
        sys.stderr.write("\n%s: the GFF3 annotation %s does not exist!\n" % ("--spliced_bam" if args.spliced_bam else "--transcript_bam", gff3))
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
                        ir_files={"markov": args.ir_markov_model, "gff3": args.ir_gff3}, ref_on_host=_plain_error_profile(args),
                        spliced=args.spliced_bam, transcript=args.transcript_bam)
    mapped_refs = None
    if args.spliced_bam:
        prof.engine.set_splice(prof.splice)
        mapped_refs = prof.spliced_refs
        _set_aln_tags(args, prof, mapped_refs)
    elif args.transcript_bam:
        mapped_refs = _transcript_refs(prof)
        if prof.ir is not None:
            prof.engine.set_splice(prof.splice)
        _set_aln_tags(args, prof, mapped_refs)
    if args.coverage is not None:
        number[0] = coverage_to_reads(prof, prof.tables.cm, args.coverage)
        prof.number_aligned, prof.number_unaligned = prof.tables.split_counts(number[0], args.perfect)
    max_len = min(max_len, prof.max_chrom)
    simulation(prof, "transcriptome", args.output, "transcriptome", args.perfect, args.KmerBias if args.homopolymer else None,
               args.basecaller, max_len, min_len, max(args.num_threads, 1), args.fastq, None, None, model_ir, args.uracil,
               args.polya, batch_reads=args.batch_reads, error_profile=not args.no_error_profile, rank=rank, world=world,
               gzip=args.gzip, gzip_error_profile=args.gzip_error_profile, bam=args.bam, mapped_refs=mapped_refs,
               transcript_bam=args.transcript_bam)
    if world > 1:
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("gloo")
        dist.barrier()
        if rank == 0:
            merge_rank_files(args.output, args.fastq, args.perfect, world, gzip=args.gzip,
                             gzip_error_profile=args.gzip_error_profile, bam=args.bam, mapped_refs=mapped_refs)
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
    mapped_refs = _mapped_refs(args, prof, False)
    _set_aln_tags(args, prof, mapped_refs)
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
                   gzip_error_profile=args.gzip_error_profile, bam=args.bam, mapped_refs=mapped_refs)
        if world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                dist.init_process_group("gloo")
            dist.barrier()
            if rank == 0:
                merge_rank_files(args.output + "_sample%d" % s_idx, args.fastq, args.perfect, world, gzip=args.gzip,
                                 gzip_error_profile=args.gzip_error_profile, bam=args.bam, mapped_refs=mapped_refs)
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


def _transcript_refs(prof):
    """--transcript_bam: bam_refs of the transcript records (the first prof.n_trx of the resident reference with intron
    retention, which puts the genome behind them, else all of them); a repeated name is a usage error."""
    ref = prof.ref
    n = prof.n_trx or len(ref.names)
    try:
        return bam_refs(_RemoteReference(ref.names[:n], np.asarray(ref.offsets)[:n + 1], ref.raw_names[:n]))
    except ValueError as e:
        sys.stderr.write("\n--transcript_bam: %s!\n" % e)
        sys.exit(1)


def _mapped_refs(args, prof, circular):
    """--mapped_bam: bam_refs of the resident reference (of the haploid one with --lift_mapped_bam), None without the flag;
    a repeated name is a usage error."""
    if not args.mapped_bam:
        return None
    try:
        return bam_refs(prof.haploid if getattr(args, "lift_mapped_bam", False) else prof.ref, circular)
    except ValueError as e:
        sys.stderr.write("\n--mapped_bam: %s!\n" % e)
        sys.exit(1)


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
    elif args.mapped_bam and args.mode == "transcriptome":
        usage = ("--mapped_bam is not available in transcriptome mode: reads that retain an intron lie on the genome (--spliced_bam "
                 "writes the alignments to the genome, --transcript_bam to the transcripts)")
    elif getattr(args, "spliced_bam", False) and not args.bam:
        usage = "--spliced_bam needs --bam"
    elif getattr(args, "spliced_bam", False) and not args.ref_g:
        usage = "--spliced_bam needs -rg: its records are against the genome"
    elif getattr(args, "transcript_bam", False) and not args.bam:
        usage = "--transcript_bam needs --bam"
    elif getattr(args, "transcript_bam", False) and args.spliced_bam:
        usage = "--transcript_bam and --spliced_bam both write <out>_aligned_reads.bam: give one of them (two runs with one --seed write the same reads)"
    elif args.mapped_bam and not args.bam:
        usage = "--mapped_bam needs --bam"
    elif getattr(args, "lift_mapped_bam", False) and not args.vcf:
        usage = "--lift_mapped_bam needs --vcf"
    elif getattr(args, "lift_mapped_bam", False) and not args.mapped_bam:
        usage = "--lift_mapped_bam needs --mapped_bam"
    elif args.aln_tags and args.mode == "transcriptome" and not (args.spliced_bam or args.transcript_bam):
        usage = "--aln_tags needs --spliced_bam in transcriptome mode, or --transcript_bam"
    elif args.aln_tags and args.mode != "transcriptome" and not args.mapped_bam:
        usage = "--aln_tags needs --mapped_bam"
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
    if args.vcf and args.dna_type == "circular":
        sys.stderr.write("\n--vcf cannot be combined with -dna_type circular!\n")
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
                        device=device, seed=args.seed or 0, ref_on_host=_plain_error_profile(args), vcf=args.vcf,
                        lift=args.lift_mapped_bam)
    if args.coverage is not None:
        number[0] = coverage_to_reads(prof, prof.tables.cm, args.coverage)
        prof.number_aligned, prof.number_unaligned = prof.tables.split_counts(number[0], args.perfect)
    max_len = min(max_len, prof.max_chrom)
    mapped_refs = _mapped_refs(args, prof, args.dna_type == "circular")
    _set_aln_tags(args, prof, mapped_refs)
    simulation(prof, args.mode, args.output, args.dna_type, args.perfect, args.KmerBias if args.homopolymer else None,
               None, max_len, min_len, max(args.num_threads, 1), args.fastq, args.median_len, args.sd_len,
               chimeric=args.chimeric, batch_reads=args.batch_reads, error_profile=not args.no_error_profile,
               rank=rank, world=world, gzip=args.gzip, gzip_error_profile=args.gzip_error_profile, bam=args.bam,
               mapped_refs=mapped_refs)
    if world > 1:
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("gloo")
        dist.barrier()
        if rank == 0:
            merge_rank_files(args.output, args.fastq, args.perfect, world, gzip=args.gzip,
                             gzip_error_profile=args.gzip_error_profile, bam=args.bam, mapped_refs=mapped_refs)
        dist.barrier()
    _log("Finished!")


if __name__ == "__main__":
    main()
