"""genome --vcf: the haplotypes of a VCF sample, parsed on the host (nanosim_b200/variants.py) and built in HBM
(ns_apply_variants, haplotype_kernel.cuh).

The reference implementation is ``build_haplotypes`` below: it reads the VCF line by line and splices strings.  The
parser's tables are checked against it on the CPU, the device's haplotype bytes on the GPU, and ``genome -rg R --vcf V``
must write exactly what ``genome -rg H`` writes, H being the builder's FASTA of the haplotype records."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

import parity_checks as pc
import synth
from nanosim_b200.reference_fasta import PackedReference, normalise_name
from nanosim_b200.variants import VcfError, read_vcf

HEADER = "##fileformat=VCFv4.2\n##contig=<ID=chr1>\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n"


def build_haplotypes(records, vcf_text):
    """Reference implementation: [(fasta header, bytes)] + VCF text -> [(``{key}-hap{h}``, bytes)]."""
    index = {h.split()[0]: i for i, (h, _) in enumerate(records)}
    ploidy, variants = {}, {}
    for line in vcf_text.splitlines():
        if not line or line.startswith("#"):
            continue
        f = line.split("\t")
        if f[6] not in ("PASS", "."):
            continue
        c = index[f[0]]
        gt = f[9].split(":")[f[8].split(":").index("GT")].replace("|", "/").split("/")
        ploidy[c] = len(gt)
        alts = f[4].split(",")
        for h, a in enumerate(gt):
            if a in (".", "0") or alts[int(a) - 1] == "*":
                continue
            variants.setdefault((c, h), []).append((int(f[1]) - 1, len(f[3]), alts[int(a) - 1].encode()))
    out = []
    for c, (header, seq) in enumerate(records):
        for h in range(ploidy.get(c, 2)):
            parts, prev = [], 0
            for p, n, alt in variants.get((c, h), []):
                parts += [seq[prev:p], alt]
                prev = p + n
            parts.append(seq[prev:])
            out.append(("%s-hap%d" % (normalise_name(header), h + 1), b"".join(parts)))
    return out


def splice_tables(t, ref):
    """The haplotype bytes the tables describe, spliced on the host."""
    out = []
    for h, c in enumerate(t.hap_chrom):
        seq = ref.bases[int(ref.offsets[c]):int(ref.offsets[c + 1])].tobytes()
        parts, prev = [], 0
        for j in range(int(t.var_off[h]), int(t.var_off[h + 1])):
            p = int(t.var_pos[j])
            parts += [seq[prev:p], t.alt[int(t.alt_off[j]):int(t.alt_off[j]) + int(t.alt_len[j])].tobytes()]
            prev = p + int(t.var_ref_len[j])
        parts.append(seq[prev:])
        out.append((t.names[h], b"".join(parts)))
    return out


def _write(path, text, gz=False):
    with (gzip.open(path, "wt") if gz else open(path, "w")) as f:
        f.write(text)
    return path


def _rows(*rows):
    return HEADER + "".join("\t".join(str(x) for x in r) + "\n" for r in rows)


def _row(chrom, pos, ref, alt, gt, filt="PASS", fmt="GT"):
    return (chrom, pos, ".", ref, alt, 50, filt, ".", fmt, gt)


SMALL = [("chr1 first", b"ACGTACGTACGTAAAACCCCGGGGTTTTacgtacgtNNNNACGTACGTACGTACGTACGT"),
         ("chr2", b"GGGGCCCCAAAATTTTGGGGCCCCAAAATTTT")]


def _small():
    return PackedReference.from_records(SMALL)


def _check(tmp_path, text, gz=False):
    path = _write(os.path.join(str(tmp_path), "v.vcf" + (".gz" if gz else "")), text, gz)
    ref = _small()
    t = read_vcf(path, ref)
    want = build_haplotypes(SMALL, text)
    assert splice_tables(t, ref) == want
    assert list(t.names) == [n for n, _ in want]
    assert t.lengths.tolist() == [len(s) for _, s in want]
    assert t.offsets.tolist() == np.concatenate([[0], np.cumsum([len(s) for _, s in want])]).tolist()
    return t


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_phased_and_unphased_gts(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 1, "A", "T", "0|1"), _row("chr1", 5, "A", "G", "1/0"), _row("chr1", 9, "A", "C", "1|1"),
                               _row("chr1", 13, "AAAA", "A", "1/1"), _row("chr2", 3, "G", "GTTT", "0/1")))
    assert t.names == ["chr1-hap1", "chr1-hap2", "chr2-hap1", "chr2-hap2"]
    assert t.applied.tolist() == [3, 3, 0, 1] and t.hap_chrom.tolist() == [0, 0, 1, 1]
    assert t.lengths.tolist() == [57, 57, 32, 35]


def test_multiallelic_records(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 2, "C", "G,T,CAT", "1|3"), _row("chr1", 6, "CG", "C,TT", "2/1"),
                               _row("chr2", 10, "A", "C,G", "2|2")))
    assert bytes(t.alt) == b"G" b"TT" b"CAT" b"C" b"G" b"G"


def test_missing_and_star_alleles(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 13, "AAAACC", "A", "0|1"), _row("chr1", 15, "A", "*,G", "2|1"),
                               _row("chr1", 20, "C", "T", ".|1"), _row("chr1", 22, "G", "A", "./."), _row("chr2", 1, "G", "*", "1/1")))
    assert t.applied.tolist() == [1, 2, 0, 0]


def test_haploid_gt(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 2, "C", "G", "0|1"), _row("chr2", 4, "G", "T", "1"), _row("chr2", 8, "C", "A", "0")))
    assert t.names == ["chr1-hap1", "chr1-hap2", "chr2-hap1"]


def test_filter_skips_records_unchecked(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 2, "C", "G", "1|1", filt="q10"), _row("chr1", 3, "G", "A", "1|0", filt="."),
                               _row("chrX", 3, "T", "<DEL>", "1|0", filt="LowQual"), _row("chr2", 3, "G", "A", "0|1", filt="PASS"),
                               _row("chr2", 4, "T", "A", "0|1", filt="q10;LowQual")))
    assert t.applied.tolist() == [1, 0, 0, 1] and t.skipped.tolist() == [1, 1, 1, 1]


def test_gzip_vcf_and_gt_not_first_in_format(tmp_path):
    _check(tmp_path, _rows(_row("chr1", 41, "A", "TGA", "30:1|0:5", fmt="GQ:GT:DP"), _row("chr2", 32, "T", "C", "0/1")), gz=True)


def test_variants_at_both_ends_and_adjacent(tmp_path):
    n = len(SMALL[0][1])
    _check(tmp_path, _rows(_row("chr1", 1, "ACG", "T", "1|1"), _row("chr1", 4, "T", "TTT", "1|0"), _row("chr1", 5, "A", "C", "1|1"),
                           _row("chr1", n, "T", "TACGT", "0|1"), _row("chr2", 1, "GGGGCCCCAAAATTTTGGGGCCCCAAAATTTT", "G", "1/1")))


def test_lower_case_ref_matches_and_alt_bytes_are_kept(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 29, "ACGT", "ncgT", "1|0"), _row("chr1", 37, "nnnn", "R", "0|1")))
    assert bytes(t.alt) == b"ncgTR"


@pytest.mark.parametrize("rows, line, message", [
    ([_row("chr1", 2, "C", "G", "0|1"), _row("chr1", 5, "T", "G", "0|1")], 5, "REF does not match"),
    ([_row("chr2", 30, "TTTTA", "T", "0|1")], 4, "past the end"),
    ([_row("chr1", 2, "CGTA", "C", "0|1"), _row("chr1", 4, "T", "G", "1|0"), _row("chr1", 5, "A", "T", "0|1")], 6, "overlaps"),
    ([_row("chr1", 2, "C", "<DEL>", "0|1")], 4, "symbolic"),
    ([_row("chr1", 2, "C", "G", "0|0"), _row("chr1", 3, "G", "G[chr2:5[", "1|0")], 5, "breakend"),
    ([_row("chr1", 2, "C", "G", "0|1"), _row("chr7", 3, "G", "A", "1|0")], 5, "unknown contig chr7"),
    ([_row("chr1", 2, "C", "G", "0/1"), _row("chr1", 3, "G", "A", "1", )], 5, "ploidy"),
    ([_row("chr1", 2, "C", "G", "0/1"), _row("chr1", 3, "G", "A", "30", fmt="GQ")], 5, "no GT"),
    ([_row("chr1", 2, "C", "G", "0/2")], 4, "larger than the number of ALT"),
    ([_row("chr1", 2, "C", "G", "0/1/1")], 4, "GT is not"),
])
def test_errors_name_the_line(rows, line, message, tmp_path):
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(*rows))
    with pytest.raises(VcfError) as e:
        read_vcf(path, _small())
    assert str(e.value).startswith("line %d:" % line) and message in str(e.value), str(e.value)


def test_the_first_error_in_the_file_is_reported(tmp_path):
    rows = [_row("chr1", 2, "C", "G", "0|1"), _row("chr1", 3, "G", "<INS>", "1|0"), _row("chr1", 5, "T", "G", "0|1"),
            _row("chr9", 6, "C", "A", "1|1"), _row("chr1", 4, "T", "G", "0|1")]
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(*rows))
    with pytest.raises(VcfError, match="^line 5: a haplotype takes an ALT allele that is symbolic"):
        read_vcf(path, _small())


def test_alt_bytes_must_be_nucleotide_codes(tmp_path):
    path = _write(os.path.join(str(tmp_path), "v.vcf"), _rows(_row("chr1", 2, "C", "G;X", "0|1")))
    with pytest.raises(VcfError, match="^line 4: .*not a nucleotide sequence"):
        read_vcf(path, _small())
    _check(tmp_path, _rows(_row("chr1", 2, "C", "ryKMbdhvNu", "0|1")))


def test_filtered_records_on_unknown_contigs_are_counted(tmp_path):
    t = _check(tmp_path, _rows(_row("chr1", 2, "C", "G", "0|1"), _row("chrUn", 3, "G", "A", "1|0", filt="LowQual"),
                               _row("chr1", 3, "G", "A", "1|0", filt="LowQual")))
    assert t.skipped_elsewhere == 1 and t.skipped.tolist() == [1, 1, 0, 0]


def test_adjacent_spans_are_not_an_overlap(tmp_path):
    _check(tmp_path, _rows(_row("chr1", 2, "CGTA", "C", "0|1"), _row("chr1", 4, "T", "G", "1|0"), _row("chr1", 6, "C", "G", "1|1")))


def test_no_sample_column(tmp_path):
    text = HEADER.replace("\tFORMAT\tSAMPLE", "") + "chr1\t2\t.\tC\tG\t50\tPASS\t.\n"
    with pytest.raises(VcfError, match="line 3: the VCF has no sample column"):
        read_vcf(_write(os.path.join(str(tmp_path), "v.vcf"), text), _small())


def test_vcf_with_circular_is_a_usage_error(tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(["genome", "-rg", "x.fa", "--vcf", "v.vcf", "-dna_type", "circular", "-o", os.path.join(str(tmp_path), "sim")])
    assert e.value.code == 1 and "--vcf cannot be combined with -dna_type circular" in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


@pytest.mark.parametrize("argv", [["metagenome", "-gl", "gl.tsv", "-a", "ab.tsv"], ["transcriptome", "-rt", "t.fa", "-e", "e.tsv"]])
def test_vcf_is_a_genome_option_only(argv, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(argv + ["--vcf", "v.vcf"])
    assert e.value.code == 2 and "unrecognized arguments: --vcf" in capsys.readouterr().err


def test_help_says_what_x_counts(capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit):
        simulator.main(["genome", "--help"])
    assert "-x 30 is about 15x per haplotype" in " ".join(capsys.readouterr().out.split())


def synthetic_genome(seed=5):
    """Three chromosomes and a VCF of ~10k SNVs, MNPs and indels: chrA (diploid) with lower-case and N stretches, a
    variant at POS 1 and one at its last base, adjacent variants, a 100 kb insertion and a 100 kb deletion; chrB without
    variants; chrC haploid.  Returns (records, vcf text)."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    a = synth.synth_chrom(rng, 700_000).copy()
    a[1000:6000] += 32                                           # lower case
    a[20_000:21_000] = ord("N")
    a[30_000:30_010] = np.frombuffer(b"RYKMSWacgn", dtype=np.uint8)
    records = [("chrA some description", a.tobytes()), ("chrB", synth.synth_chrom(rng, 300_000).tobytes()),
               ("chrC", synth.synth_chrom(rng, 250_000).tobytes())]
    rows = []

    def seq(n):
        return acgt[rng.integers(0, 4, n)].tobytes().decode()

    def add(chrom, pos, ref_len, alt, gt, filt="PASS"):
        s = dict((h.split()[0], b) for h, b in records)[chrom]
        rows.append(_row(chrom, pos, s[pos - 1:pos - 1 + ref_len].decode(), alt, gt, filt))

    for chrom, lo, hi, gts in (("chrA", 1, 700_000, ["0|1", "1|0", "1|1", "0/1", "1|2", "2/1"]), ("chrC", 1, 250_000, ["1", "0", "2"])):
        pos = lo
        if chrom == "chrA":
            add("chrA", 1, 1, "G", "1|1")                                # POS 1
            add("chrA", 2, 3, "T", "0|1")                                # adjacent to it
            add("chrA", 5, 1, "CC", "1|0")                               # and adjacent again
            add("chrA", 200_000, 100_000, "A", "0|1")                    # 100 kb deletion
            add("chrA", 400_000, 1, "T" + seq(100_000), "1|0")           # 100 kb insertion
            pos = 10
        while True:
            pos += int(rng.integers(1, 120))
            if chrom == "chrA" and 199_000 < pos < 401_000:
                pos = 401_000
            kind = rng.integers(0, 4)
            n = 1 if kind == 0 else int(rng.integers(2, 12))
            if pos + n >= hi - 20:
                break
            if kind == 0:
                alt = seq(1)
            elif kind == 1:
                alt = seq(n)                                             # MNP
            elif kind == 2:
                alt = seq(1)                                             # deletion
            else:
                alt, n = seq(int(rng.integers(2, 30))), 1                # insertion
            alt2 = seq(1) if "2" in "".join(gts) else None
            gt = gts[int(rng.integers(0, len(gts)))]
            add(chrom, pos, n, alt + ("," + alt2 if alt2 else ""), gt, "PASS" if rng.random() > 0.05 else "LowQual")
            pos += n - 1
        if chrom == "chrA":
            add("chrA", hi, 1, "A", "1|0")                               # last base
    rows.sort(key=lambda r: (r[0], r[1]))
    return records, HEADER + "".join("\t".join(str(x) for x in r) + "\n" for r in rows)


@pytest.fixture(scope="module")
def genome(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("vcf"))
    records, text = synthetic_genome()
    ref = os.path.join(d, "ref.fa")
    synth.write_fasta(ref, [(h, np.frombuffer(s, dtype=np.uint8)) for h, s in records])
    vcf = _write(os.path.join(d, "sample.vcf.gz"), text, gz=True)
    haps = build_haplotypes(records, text)
    hap_fa = os.path.join(d, "hap.fa")
    synth.write_fasta(hap_fa, [(n, np.frombuffer(s, dtype=np.uint8)) for n, s in haps])
    return d, ref, vcf, hap_fa, records, text, haps


def test_synthetic_tables_equal_the_builder(genome):
    d, ref, vcf, hap_fa, records, text, haps = genome
    r = PackedReference.from_fasta(ref)
    t = read_vcf(vcf, r)
    assert splice_tables(t, r) == haps
    assert t.names == ["chrA-hap1", "chrA-hap2", "chrB-hap1", "chrB-hap2", "chrC-hap1"]
    assert int(t.applied.sum()) > 8000 and t.applied[2:4].tolist() == [0, 0]
    assert max(len(s) for _, s in haps) > 700_000


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_device_haplotypes_equal_the_builder(genome):
    from nanosim_b200.engine import Engine, NanoSimError
    d, ref, vcf, hap_fa, records, text, haps = genome
    r = PackedReference.from_fasta(ref)
    t = read_vcf(vcf, r)
    eng = Engine(device=0, seed=1)
    with pytest.raises(NanoSimError, match="set the reference first"):
        eng.apply_variants(t)
    eng.set_reference(r)
    peak = eng.apply_variants(t)
    want = b"".join(s for _, s in haps)
    assert eng.reference_bases(len(want)).tobytes() == want
    assert peak >= 2 * len(want)
    clone = eng.clone()
    with pytest.raises(NanoSimError, match="cloned context"):
        clone.apply_variants(t)
    clone.close()
    eng.close()


_E2E = {
    "guppy_fastq": ["-c", "guppy", "-n", "3000", "--fastq", "--seed", "41"],
    "dorado_hp6_chimeric": ["-c", "dorado", "-n", "2000", "--fastq", "-hp", "-k", "6", "--chimeric", "--seed", "42"],
    "gzip_gzip_error_profile": ["-c", "guppy", "-n", "3000", "--fastq", "--gzip", "--gzip_error_profile", "--seed", "43"],
    "bam": ["-c", "guppy", "-n", "3000", "--fastq", "--bam", "--seed", "44"],
    "guppy_fasta_batch_reads": ["-c", "guppy", "-n", "3000", "--seed", "41", "--batch_reads", "700"],
}


def _argv(extra):
    extra = list(extra)
    extra[1] = os.path.join(pc.DATA, pc.MODELS[extra[1]])
    return extra + ["-t", "4"]


def _outputs(prefix):
    d, base = os.path.split(prefix)
    return sorted(f[len(base):] for f in os.listdir(d) if f.startswith(base + "_"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_E2E))
def test_vcf_run_equals_a_run_on_the_haplotype_fasta(name, genome):
    from nanosim_b200 import simulator
    d, ref, vcf, hap_fa, records, text, haps = genome
    a, b = os.path.join(d, name + "_vcf"), os.path.join(d, name + "_hap")
    simulator.main(["genome", "-rg", ref, "--vcf", vcf, "-o", a] + _argv(_E2E[name]))
    simulator.main(["genome", "-rg", hap_fa, "-o", b] + _argv(_E2E[name]))
    files = _outputs(a)
    assert files == _outputs(b) and len(files) >= 3, files
    for f in files:
        x, y = open(a + f, "rb").read(), open(b + f, "rb").read()
        assert x == y and len(x) > 1000, f
    if name == "guppy_fastq":
        reads = open(a + "_aligned_reads.fastq", "rb").read()
        assert b"@chrA-hap2_" in reads and b"@chrC-hap1_" in reads


@pytest.mark.gpu
def test_vcf_run_is_independent_of_batching(genome):
    from nanosim_b200 import simulator
    d, ref, vcf, hap_fa, records, text, haps = genome
    a, b = os.path.join(d, "batch_a"), os.path.join(d, "batch_b")
    simulator.main(["genome", "-rg", ref, "--vcf", vcf, "-o", a] + _argv(_E2E["guppy_fastq"]))
    simulator.main(["genome", "-rg", ref, "--vcf", vcf, "-o", b, "--batch_reads", "512"] + _argv(_E2E["guppy_fastq"]))
    for f in _outputs(a):
        assert open(a + f, "rb").read() == open(b + f, "rb").read(), f


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(genome):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    d, ref, vcf, hap_fa, records, text, haps = genome
    args = ["genome", "-rg", ref, "--vcf", vcf] + _argv(_E2E["guppy_fastq"]) + ["--batch_reads", "700"]
    one, two = os.path.join(d, "ranks_one"), os.path.join(d, "ranks_two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29747", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.fastq", "_unaligned_reads.fastq", "_aligned_error_profile"):
        x, y = open(one + f, "rb").read(), open(two + f, "rb").read()
        assert x == y and len(x) > 1000, f
