"""The emit kernel's output bytes, pinned across builds: SHA-256 of the bases and the qualities of fixed-seed batches that
reach every branch of emit_kernel.cuh (fast and exact route, forward and reverse reads, aligned and unaligned batches,
circular wrap-around, IUPAC and lower-case reference bytes, minus-strand retained-intron pieces, split and whole pieces
longer than 40 kb, FASTQ and FASTA).  The other tests compare one route or one split with another in the same build; this
one fails when a change to the kernel changes any byte it writes.

`python tests/test_emit_bytes.py` prints the digests of the current build in the layout of DIGESTS."""
import hashlib
import os
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conftest import GOLDEN  # noqa: E402

import parity_checks as pc  # noqa: E402
import synth  # noqa: E402

ALIGNED, UNALIGNED = 0, 1

# case -> (sha256 of the bases, sha256 of the qualities) of every read of the case's batches, in batch order
DIGESTS = {
    "guppy_fastq": ("acf246488f5486c9858d6d89f2d4f41161e027f9557394f2769209003dec6bfd",
        "6dfb999975e12890eaf03ed78fe711b76d7839785bd51e5c84822e9f651fc86a"),
    "guppy_fasta": ("874810e9d6995ad430dfcf0ff0b0a26fc1be85eb76610735bc334971d6a27700",
        "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"),
    "guppy_fastq_exact": ("acf246488f5486c9858d6d89f2d4f41161e027f9557394f2769209003dec6bfd",
        "6dfb999975e12890eaf03ed78fe711b76d7839785bd51e5c84822e9f651fc86a"),
    "guppy_fastq_whole": ("acf246488f5486c9858d6d89f2d4f41161e027f9557394f2769209003dec6bfd",
        "6dfb999975e12890eaf03ed78fe711b76d7839785bd51e5c84822e9f651fc86a"),
    "guppy_fastq_circular": ("c353e107545a1aba2971f25fbe8e8a771ea1a6be73e13677d62eebec32a05d34",
        "6dfb999975e12890eaf03ed78fe711b76d7839785bd51e5c84822e9f651fc86a"),
    "dorado_chimeric": ("cfcf833dd13ee5f8a2c9ebaf8db0f498fe304a9c517c13e00c40e0271a8a3b6f",
        "d70eda3195b9d22d2b97ef4c1e97f44daccae8d1c70f5c289a69e0557f4569ad"),
    "dorado_chimeric_fasta": ("e2618ee8b4511bbb0dda960c4e8f675fab37ec701e60f87bcc79f1fba45cf75e",
        "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"),
    "dorado_hp6": ("5535571bbfd59d384bf0e761d816294d7303ad93247bf93080e3a4f15301fc5a",
        "cc52b1c2693b273645fd2e43d3127030395544d7937403bdb7488d592f5e2c6a"),
    "mini_ref_fastq": ("d8bb25f637cd5967c9e81dcd041bd6bf25f911aaea52f11d3dc749aca03db796",
        "e1ad75986b8a579002eacb2092702917226a82d17d07dff7a8313982e63cdb64"),
    "mini_ref_fasta": ("67e36d418634450635581f62e1061bad8d6a9a7813e674aa8bc0b7c5135242e3",
        "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"),
    "ir_minus_strand_polya_hp6": ("9c16dba6d7c6763822e40fe5980500537ae2d44f0bc5ab2b015858306f65365b",
        "81a9c13c6d46904af5958b49a5e95771b7349fff11579643884ebb15a8e512ac"),
}

# case -> (model, reference, engine keywords); every case runs an aligned and an unaligned batch
GENOME_CASES = {
    "guppy_fastq": ("guppy", "ecoli", dict(fastq=True)),
    "guppy_fasta": ("guppy", "ecoli", dict(fastq=False)),
    "guppy_fastq_exact": ("guppy", "ecoli", dict(fastq=True, emit_exact=True)),
    "guppy_fastq_whole": ("guppy", "ecoli", dict(fastq=True, emit_whole=True)),
    "guppy_fastq_circular": ("guppy", "ecoli", dict(fastq=True, circular=True)),
    "dorado_chimeric": ("dorado", "ecoli", dict(fastq=True, chimeric=True)),
    "dorado_chimeric_fasta": ("dorado", "ecoli", dict(fastq=False, chimeric=True)),
    "dorado_hp6": ("dorado", "ecoli", dict(fastq=True, chimeric=True, kmer_bias=6)),
    "mini_ref_fastq": ("guppy", "mini_ref", dict(fastq=True)),
    "mini_ref_fasta": ("guppy", "mini_ref", dict(fastq=False)),
}


class _Digest:
    def __init__(self):
        self.seq, self.qual = hashlib.sha256(), hashlib.sha256()

    def add(self, b, fastq):
        for r in b.reads:
            a, n = int(r["seq_off"]), int(r["seq_len"])
            self.seq.update(b.seq[a:a + n].tobytes())
            if fastq:
                self.qual.update(b.qual[a:a + n].tobytes())

    def hex(self):
        return self.seq.hexdigest(), self.qual.hexdigest()


def _references():
    from nanosim_b200.reference_fasta import PackedReference
    return {"ecoli": PackedReference.from_records(synth.ecoli5m()),
            "mini_ref": PackedReference.from_fasta(os.path.join(GOLDEN, "mini_ref.fa"))}


def genome_digest(name, refs):
    model, ref, kw = GENOME_CASES[name]
    eng, _, _ = pc.make_engine(model, refs[ref], seed=4242, **kw)
    d = _Digest()
    n_long = 0
    for kind, first, n in ((ALIGNED, 17, 3000), (UNALIGNED, 9, 1500)):
        eng.simulate(kind, first, n)
        b = eng.fetch(want_ops=True)
        d.add(b, kw.get("fastq", False))
        n_long += int((b.pieces["out_len"] > 40000).sum())
        rev = b.reads["reversed"] != 0
        assert rev.any() and (~rev).any()
    eng.close()
    if ref == "ecoli":
        assert n_long > 0, "no piece longer than 40 kb: the split is not exercised"
    return d.hex()


def ir_digest():
    """Transcriptome reads with polyA tails whose retained introns are re-emitted on the genome, minus-strand pieces
    (NS_PIECE_REF_REV) with IUPAC and lower-case intron bytes among them, -hp -k 6 (the fixture of test_ir_homopolymer)."""
    import test_ir_homopolymer as irh
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.reference_fasta import PackedReference, read_expression, read_polya_list
    with tempfile.TemporaryDirectory() as d:
        irh._write_fixture(d)
        model, cm = irh._hp_model(d)
        trx = PackedReference.from_fasta(os.path.join(d, "transcripts.fa"))
        genome = PackedReference.from_fasta(os.path.join(d, "genome.fa"))
        ref = PackedReference.concat(trx, genome)
        chrom, w = read_expression(os.path.join(d, "expression.tsv"), trx)
        polya = np.concatenate([read_polya_list(os.path.join(d, "polya.txt"), trx), np.zeros(len(genome.names), dtype=np.uint8)])
        st = ir.TranscriptStructures.from_gff3(os.path.join(d, "annotation.gff3"), trx.names, genome.raw_names)
        irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(d, "IR_markov_model")), st, trx.lengths, len(trx.names))
        fx = dict(cm=cm, ref=ref, chrom=chrom, w=w, polya=polya, trx=trx)
        eng = irh._engine(fx, 6, 77)
        _, _, patch, b1 = irh._simulate_and_retain(eng, irm, 500, 4000, 77)
        minus = (b1.pieces["kind"].astype(np.int64) & L.NS_PIECE_REF_REV) != 0
        assert len(patch[0]) > 0 and minus.any()
        d_ = _Digest()
        d_.add(b1, True)
        eng.close()
    return d_.hex()


@pytest.fixture(scope="module")
def refs():
    return _references()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GENOME_CASES))
def test_emit_bytes_genome(name, refs):
    assert genome_digest(name, refs) == DIGESTS[name]


@pytest.mark.gpu
def test_emit_bytes_ir_minus_strand():
    assert ir_digest() == DIGESTS["ir_minus_strand_polya_hp6"]


if __name__ == "__main__":
    r = _references()
    out = {name: genome_digest(name, r) for name in sorted(GENOME_CASES)}
    out["ir_minus_strand_polya_hp6"] = ir_digest()
    for k, (s, q) in out.items():
        print('    "%s": ("%s",\n        "%s"),' % (k, s, q))
