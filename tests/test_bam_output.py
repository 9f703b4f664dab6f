"""--bam: the reads as unaligned BAM, encoded and BGZF-compressed on the GPU (ns_compress_bam).

Decompressed, every .bam file must be the BAM header followed by one unmapped record per read of the plain FASTA/FASTQ
file of the same run, in the same order, as the Python encoder below writes it; each member must be a valid BGZF member
whose Huffman code is close to optimal.  pysam and samtools are not needed: the reader and the encoder are here.  GPU
tests run with ``pytest -m gpu``; the CLI, header and rank-merge tests at the end need no GPU."""
import ctypes
import gzip
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

import parity_checks as pc
import synth
from test_bgzf_output import BLOCK, _EmptyPipeline, _empty_profile, _zlib_member, bgzf_members, check_bgzf_file

SAM_CODES = "=ACMGRSVTWYHKDBN"          # SAM/BAM specification §4.2.3: 4-bit base codes
_CODE = np.full(256, 15, dtype=np.uint8)
for _k, _c in enumerate(SAM_CODES):
    _CODE[ord(_c)] = _CODE[ord(_c.lower())] = _k
_CODE[ord("U")] = _CODE[ord("u")] = _CODE[ord("T")]  # as htslib reads it


def _eof():
    from nanosim_b200.simulator import BGZF_EOF
    return BGZF_EOF


def header_bytes():
    """The decompressed BAM header the simulator writes."""
    from nanosim_b200.simulator import bam_header
    return gzip.decompress(bam_header())


def bam_record(name, seq, qual):
    """One unmapped BAM record as the specification lays it out; qual None: a FASTA read (0xff qualities)."""
    L = len(seq)
    codes = _CODE[np.frombuffer(seq, dtype=np.uint8)]
    if L % 2:
        codes = np.append(codes, np.uint8(0))
    packed = ((codes[0::2] << 4) | codes[1::2]).astype(np.uint8).tobytes()
    q = b"\xff" * L if qual is None else (np.frombuffer(qual, dtype=np.uint8) - 33).astype(np.uint8).tobytes()
    body = struct.pack("<iiBBHHHIiii", -1, -1, len(name) + 1, 255, 4680, 0, 4, L, -1, -1, 0) + name + b"\0" + packed + q
    return struct.pack("<i", len(body)) + body


def parse_records(text, fastq):
    """(name, seq, qual) of every record of the simulator's FASTA/FASTQ text (one line per field)."""
    lines = text.split(b"\n")
    assert lines[-1] == b""
    k = 4 if fastq else 2
    assert (len(lines) - 1) % k == 0
    return [(lines[i][1:], lines[i + 1], lines[i + 3] if fastq else None) for i in range(0, len(lines) - 1, k)]


def encode_text(text, fastq):
    return b"".join(bam_record(n, s, q) for n, s, q in parse_records(text, fastq))


def read_bam(data):
    """(header text, records) of a decompressed BAM file: every record as a dict of its fields."""
    assert data[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", data, 4)[0]
    text = data[8:8 + l_text]
    pos = 8 + l_text
    assert struct.unpack_from("<i", data, pos)[0] == 0                # n_ref
    pos += 4
    recs = []
    while pos < len(data):
        block, ref_id, p, l_name, mapq, bin_, n_cig, flag, l_seq, nref, npos, tlen = struct.unpack_from("<iiiBBHHHIiii", data, pos)
        q = pos + 36
        name = data[q:q + l_name]
        assert name[-1:] == b"\0"
        q += l_name
        packed = np.frombuffer(data, dtype=np.uint8, count=(l_seq + 1) // 2, offset=q)
        codes = np.empty(2 * len(packed), dtype=np.uint8)
        codes[0::2], codes[1::2] = packed >> 4, packed & 15
        q += (l_seq + 1) // 2
        qual = data[q:q + l_seq]
        assert q + l_seq == pos + 4 + block, "record at %d: block_size %d" % (pos, block)
        recs.append(dict(name=name[:-1], ref_id=ref_id, pos=p, mapq=mapq, bin=bin_, n_cigar=n_cig, flag=flag, l_seq=l_seq,
                         next_ref_id=nref, next_pos=npos, tlen=tlen, codes=codes[:l_seq], pad=codes[l_seq:], qual=qual))
        pos += 4 + block
    assert pos == len(data)
    return text, recs


def check_bam_file(path):
    """BGZF structure of a .bam file (see check_bgzf_file), the header alone in the first member; its decompressed bytes."""
    data = check_bgzf_file(path)
    first = bgzf_members(open(path, "rb").read())[0]
    assert first[2] == len(header_bytes()) and data.startswith(header_bytes()), path
    return data


# ---------------------------------------------------------------------------------------------------------------- GPU
_CONFIGS = ["genome_fastq_chimeric", "genome_fasta", "dorado_fastq_hp6", "metagenome_chimeric", "transcriptome_ir"]
_RUNS = {}


def _ecoli(tmp):
    ref = os.path.join(tmp, "ecoli5m.fa")
    if not os.path.exists(ref):
        synth.ecoli5m(ref)
    return ref


def _guppy():
    return os.path.join(pc.DATA, pc.MODELS["guppy"])


def _config_args(name, tmp):
    """(command line, fastq) of a configuration (those of test_bgzf_output, the transcriptome one without --uracil)."""
    from conftest import meta_fixture
    ref = _ecoli(tmp)
    if name == "genome_fastq_chimeric":
        return ["genome", "-rg", ref, "-c", _guppy(), "-n", "2500", "--fastq", "--chimeric", "--seed", "21"], True
    if name == "genome_fasta":
        return ["genome", "-rg", ref, "-c", _guppy(), "-n", "2500", "--seed", "22"], False
    if name == "dorado_fastq_hp6":
        return ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["dorado"]), "-n", "2000", "--fastq", "-hp", "-k", "6",
                "--chimeric", "--seed", "23"], True
    if name == "metagenome_chimeric":
        meta_fixture()                                          # writes genome_list_local.tsv
        M = os.path.join(GOLDEN, "meta")
        return ["metagenome", "-gl", os.path.join(M, "genome_list_local.tsv"), "-a", os.path.join(M, "abundance.tsv"), "-dl",
                os.path.join(M, "dna_type.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["even"]), "--fastq", "--chimeric", "--seed", "24"], True
    D = os.path.join(GOLDEN, "ir")
    return ["transcriptome", "-rt", os.path.join(D, "transcripts.fa"), "-rg", os.path.join(D, "genome.fa"), "-e",
            os.path.join(D, "expression.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", "1500",
            "--polya", os.path.join(D, "polya.txt"), "-b", "guppy", "--seed", "25", "--batch_reads", "600",
            "--ir_markov_model", os.path.join(D, "IR_markov_model"), "--ir_gff3", os.path.join(D, "annotation.gff3")], False


def _run_config(name, tmp):
    """Runs the configuration once plain and once with --bam (same seed): (plain prefix, bam prefix, fastq, sample
    prefixes)."""
    from nanosim_b200 import simulator
    if name not in _RUNS:
        args, fastq = _config_args(name, tmp)
        plain, bam = os.path.join(tmp, name + "_plain"), os.path.join(tmp, name + "_bam")
        simulator.main(args + ["-o", plain, "-t", "4"])
        simulator.main(args + ["-o", bam, "-t", "4", "--bam"])
        _RUNS[name] = (plain, bam, fastq, ["_sample0", "_sample1"] if name == "metagenome_chimeric" else [""])
    return _RUNS[name]


@pytest.fixture(scope="module")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("bam"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_bam_equals_the_encoded_plain_records(name, workdir):
    plain, bam, fastq, samples = _run_config(name, workdir)
    ext = ".fastq" if fastq else ".fasta"
    for p in samples:
        recs = []
        for f in ("_aligned_reads", "_unaligned_reads"):
            text = open(plain + p + f + ext, "rb").read()
            assert len(text) > 1000 and not os.path.exists(bam + p + f + ext) and not os.path.exists(bam + p + f + ext + ".gz")
            data = gzip.decompress(open(bam + p + f + ".bam", "rb").read())
            assert data == header_bytes() + encode_text(text, fastq), f
            recs += read_bam(data)[1]
        err = p + "_aligned_error_profile"
        assert open(plain + err, "rb").read() == open(bam + err, "rb").read(), err
        assert any(r["l_seq"] % 2 for r in recs) and all(r["flag"] == 4 for r in recs)
        assert any(b"_R_" in r["name"] for r in recs) and any(b"_F_" in r["name"] for r in recs)
    if name == "transcriptome_ir":                             # these batches went through ns_reemit
        assert any(b"_RetainedIntron_" in r["name"] for r in recs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_bam_members_are_valid_and_near_optimal(name, workdir):
    plain, bam, fastq, samples = _run_config(name, workdir)
    ext = ".fastq" if fastq else ".fasta"
    for p in samples:
        for f in ("_aligned_reads", "_unaligned_reads"):
            data = check_bam_file(bam + p + f + ".bam")
            assert data == header_bytes() + encode_text(open(plain + p + f + ext, "rb").read(), fastq)


@pytest.mark.gpu
def test_gzip_error_profile_with_bam(workdir):
    from nanosim_b200 import simulator
    plain, _, _, _ = _run_config("genome_fastq_chimeric", workdir)
    args, _ = _config_args("genome_fastq_chimeric", workdir)
    out = os.path.join(workdir, "bam_gzerr")
    simulator.main(args + ["-o", out, "-t", "4", "--bam", "--gzip_error_profile"])
    assert not os.path.exists(out + "_aligned_error_profile")
    want = open(plain + "_aligned_error_profile", "rb").read()
    assert gzip.decompress(open(out + "_aligned_error_profile.gz", "rb").read()) == want and len(want) > 1000
    text = open(plain + "_aligned_reads.fastq", "rb").read()
    assert gzip.decompress(open(out + "_aligned_reads.bam", "rb").read()) == header_bytes() + encode_text(text, True)


@pytest.mark.gpu
def test_bam_is_independent_of_batching(tmp_path):
    from nanosim_b200 import simulator
    ref = _ecoli(str(tmp_path))
    outs = []
    for batch in (["--batch_reads", "700"], []):
        out = os.path.join(str(tmp_path), "b%d" % len(batch))
        simulator.main(["genome", "-rg", ref, "-c", _guppy(), "-n", "4000", "--fastq", "--seed", "34", "-t", "3", "--bam", "-o", out] + batch)
        outs.append(out)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        a, b = (check_bam_file(o + f) for o in outs)
        assert a == b and len(read_bam(a)[1]) > 100, f


@pytest.fixture(scope="module")
def ecoli():
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_records(synth.ecoli5m())


def _bam_batch(eng, ref, kind, n, first=0):
    """Simulates one batch, formats it on the host and compresses it as BAM on the device: (encoded records, members)."""
    from nanosim_b200.records import format_records, name_table
    eng.simulate(kind, first, n)
    b = eng.fetch()
    names = name_table(b, ref.names, first)
    want = encode_text(format_records(b, names, eng.fastq), eng.fastq)
    nz = eng.compress_bam(names)
    members = eng.fetch_compressed().tobytes()
    assert len(members) == nz
    return want, members, names


@pytest.mark.gpu
def test_engine_one_read_capacity_and_state(ecoli):
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import NanoSimError
    from nanosim_b200.engine import _ptr
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=True, seed=31)
    n, offs = ctypes.c_uint64(), np.zeros(1, dtype=np.uint64)
    with pytest.raises(NanoSimError, match="no simulated batch.*rc=-3"):
        eng._check(eng._lib.ns_compress_bam(eng._ctx, b"r\0", _ptr(offs), ctypes.byref(n)))
    want, members, names = _bam_batch(eng, ecoli, L.NS_KIND_ALIGNED, 1)
    assert len(bgzf_members(members)) == 1 and gzip.decompress(members + _eof()) == want
    assert eng.compress_bam(names) == len(members) and eng.fetch_compressed().tobytes() == members     # deterministic
    with pytest.raises(NanoSimError, match="rc=-4"):
        eng.fetch_compressed(np.empty(len(members) - 1, dtype=np.uint8))
    # the records compression and the BAM one replace each other's members
    nr = eng.compress_records(names)
    assert gzip.decompress(eng.fetch_compressed().tobytes() + _eof()).startswith(b"@")
    assert eng.compress_bam(names) == len(members) != nr and eng.fetch_compressed().tobytes() == members
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fastq", [False, True])
def test_records_longer_than_several_blocks(ecoli, fastq, tmp_path):
    from nanosim_b200 import _lib as L
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=fastq, seed=32)
    eng.configure(fastq=fastq, min_len=200000, max_len=ecoli.max_chrom, median_len=300000, sd_len=0.1)
    want, members, _ = _bam_batch(eng, ecoli, L.NS_KIND_ALIGNED, 5)
    assert eng.info.total_bases / 5 > 3 * BLOCK
    path = os.path.join(str(tmp_path), "long.bam")
    with open(path, "wb") as f:
        f.write(members + _eof())
    assert check_bgzf_file(path) == want
    recs = read_bam(header_bytes() + want)[1]
    assert len(recs) == 5 and all(r["qual"] == b"\xff" * r["l_seq"] for r in recs) != fastq
    eng.close()


@pytest.mark.gpu
def test_name_lengths_and_bytes_above_0x7f(ecoli):
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import NanoSimError
    from nanosim_b200.records import format_records
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=True, seed=36)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 3)
    b = eng.fetch()
    names = ["r" * 254, "read_éß中_1", "x"]
    eng.compress_bam(names)
    got = gzip.decompress(eng.fetch_compressed().tobytes() + _eof())
    assert got == encode_text(format_records(b, names, True), True)
    assert [r["name"] for r in read_bam(header_bytes() + got)[1]] == [n.encode() for n in names]
    with pytest.raises(NanoSimError, match=r"read 1 has a name of 255 bytes.*rc=-1"):
        eng.compress_bam(["a", "b" * 255, "c" * 300])
    eng.close()


@pytest.mark.gpu
def test_iupac_lower_case_and_other_bytes(tmp_path):
    """A reference with IUPAC codes, lower case and a byte that is no nucleotide code (J): the BAM bases are the 4-bit codes
    of the FASTA output's bases.  case_convert resolves the IUPAC codes, and the emit kernel writes every base through its
    2-bit index, so the reads hold A C G T only; test_every_byte_value_is_coded gives the kernel the other bytes."""
    from nanosim_b200 import simulator
    rng = np.random.default_rng(5)
    seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, 300000)].copy()
    odd = np.frombuffer(b"RYKMSWBDHVNXacgtryknx" + b"Jj" * 4, dtype=np.uint8)
    at = rng.choice(len(seq), 6000, replace=False)
    seq[at] = odd[rng.integers(0, len(odd), len(at))]
    ref = os.path.join(str(tmp_path), "iupac.fa")
    synth.write_fasta(ref, [("chrI", seq)])
    args = ["genome", "-rg", ref, "-c", _guppy(), "-n", "600", "--seed", "37"]
    plain, bam = os.path.join(str(tmp_path), "p"), os.path.join(str(tmp_path), "b")
    simulator.main(args + ["-o", plain])
    simulator.main(args + ["-o", bam, "--bam"])
    text = open(plain + "_aligned_reads.fasta", "rb").read()
    recs = read_bam(check_bam_file(bam + "_aligned_reads.bam"))[1]
    seqs = [s for _, s, _ in parse_records(text, False)]
    assert len(recs) == len(seqs) > 100 and set(b"".join(seqs)) == set(b"ACGT")
    for r, s in zip(recs, seqs):
        assert r["l_seq"] == len(s) and (r["codes"] == _CODE[np.frombuffer(s, dtype=np.uint8)]).all() and not r["pad"].any()


@pytest.mark.gpu
def test_every_byte_value_is_coded(ecoli):
    """Every byte value in the device's sequence buffer, as the BAM kernel reads it: the SAM codes of both cases, U as T,
    and N (15) for the 256 - 33 other bytes.  The bytes are written over the first read's bases in HBM."""
    import torch
    from nanosim_b200 import _lib as L
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=True, seed=38)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 4)
    b = eng.fetch()
    r0 = b.reads[int(np.argmax(b.reads["seq_len"]))]
    o, n = int(r0["seq_off"]), int(r0["seq_len"])
    assert n >= 256
    pattern = (np.arange(n) % 256).astype(np.uint8)

    class _Span:                        # the read's bytes in HBM, as a torch tensor aliases them
        __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "version": 2,
                                    "data": (eng.device_buffers()["seq"] + o, False)}
    torch.as_tensor(_Span(), device="cuda").copy_(torch.from_numpy(pattern))
    torch.cuda.synchronize()
    b.seq[o:o + n] = pattern
    names = ["r%d" % i for i in range(4)]
    eng.compress_bam(names)
    got = gzip.decompress(eng.fetch_compressed().tobytes() + _eof())
    seqs = [b.seq[int(r["seq_off"]):int(r["seq_off"]) + int(r["seq_len"])].tobytes() for r in b.reads]
    quals = [b.qual[int(r["seq_off"]):int(r["seq_off"]) + int(r["seq_len"])].tobytes() for r in b.reads]
    assert got == b"".join(bam_record(nm.encode(), s, q) for nm, s, q in zip(names, seqs, quals))
    rec = [r for r in read_bam(header_bytes() + got)[1] if r["l_seq"] == n][0]
    codes = rec["codes"][:256]
    assert (codes == _CODE).all()
    assert [codes[ord(c)] for c in "=aAcCgGtTuUnNJj*"] == [0, 1, 1, 2, 2, 4, 4, 8, 8, 8, 8, 15, 15, 15, 15, 15]
    assert codes[0] == codes[0xff] == codes[ord("\n")] == 15
    eng.close()


@pytest.mark.gpu
def test_after_reemit():
    """ns_compress_bam after ns_reemit (reads that retain an intron are emitted again on the genome): the records are
    those of the patched batch."""
    from nanosim_b200 import _lib as L
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.records import format_records, name_table
    from nanosim_b200.reference_fasta import POLYA_SCALE, PackedReference, read_expression, read_polya_list
    D = os.path.join(GOLDEN, "ir")
    trx = PackedReference.from_fasta(os.path.join(D, "transcripts.fa"))
    genome = PackedReference.from_fasta(os.path.join(D, "genome.fa"))
    ref = PackedReference.concat(trx, genome)
    chrom, w = read_expression(os.path.join(D, "expression.tsv"), trx)
    polya = np.concatenate([read_polya_list(os.path.join(D, "polya.txt"), trx), np.zeros(len(genome.names), dtype=np.uint8)])
    st = ir.TranscriptStructures.from_gff3(os.path.join(D, "annotation.gff3"), trx.names, genome.raw_names)
    irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(D, "IR_markov_model")), st, trx.lengths, len(trx.names))
    eng, _, _ = pc.make_trx_engine(ref, chrom, w, polya, fastq=True, seed=39, polya_scale=POLYA_SCALE["guppy"],
                                   trx_records=len(trx.names), max_len=trx.max_chrom)
    eng.simulate(L.NS_KIND_ALIGNED, 500, 800)
    b0 = eng.fetch(want_ops=True)
    eng.compress_bam(name_table(b0, ref.names, 500, transcriptome=True))
    patch = irm.plan_batch(b0.reads, b0.pieces, b0.ops, 500, 39, eng.info.n_pieces, eng.info.n_ops)
    assert patch is not None
    eng.reemit(*patch)
    b1 = eng.fetch()
    names = name_table(b1, ref.names, 500, transcriptome=True)
    eng.compress_bam(names)
    got = gzip.decompress(eng.fetch_compressed().tobytes() + _eof())
    assert got == encode_text(format_records(b1, names, True), True)
    assert b"_RetainedIntron_" in got
    eng.close()


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = _ecoli(str(tmp_path))
    args = ["genome", "-rg", ref, "-c", _guppy(), "-n", "4000", "--fastq", "--seed", "35", "--batch_reads", "700", "-t", "4", "--bam"]
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29745", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.bam", "_unaligned_reads.bam"):
        assert check_bam_file(two + f) == check_bam_file(one + f), f
    assert not os.path.exists(two + "_aligned_reads1.bam")


# ---------------------------------------------------------------------------------------------------------------- CPU
_ARGV = {"genome": ["genome", "-rg", "x.fa"], "metagenome": ["metagenome", "-gl", "gl.tsv", "-a", "ab.tsv"],
         "transcriptome": ["transcriptome", "-rt", "t.fa", "-e", "e.tsv", "--no_model_ir"]}


@pytest.mark.parametrize("mode, extra, message", [
    ("genome", ["--bam", "--gzip"], "--bam and --gzip"),
    ("metagenome", ["--bam", "--gzip"], "--bam and --gzip"),
    ("transcriptome", ["--bam", "--uracil"], "--bam cannot be combined with --uracil"),
    ("genome", ["--gzip_error_profile"], "--gzip_error_profile needs --gzip"),
    ("transcriptome", ["--gzip_error_profile"], "--gzip_error_profile needs --gzip or --bam"),
])
def test_usage_errors(mode, extra, message, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV[mode] + ["-o", os.path.join(str(tmp_path), "sim")] + extra)
    assert e.value.code == 1
    assert message in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


@pytest.mark.parametrize("mode", list(_ARGV))
@pytest.mark.parametrize("fastq", [False, True])
def test_bam_flag_names_the_outputs(mode, fastq, tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    monkeypatch.setattr(simulator, "read_profile", _empty_profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(_ARGV[mode] + ["-o", out, "--bam"] + (["--fastq"] if fastq else []))
    prefix = out + ("_sample0" if mode == "metagenome" else "")
    for f in ("_aligned_reads", "_unaligned_reads"):
        assert open(prefix + f + ".bam", "rb").read() == simulator.bam_header() + _eof()
        for ext in (".fasta", ".fastq", ".fasta.gz", ".fastq.gz"):
            assert not os.path.exists(prefix + f + ext)
    assert open(prefix + "_aligned_error_profile").read().startswith("Seq_name\t")


def test_header_parses_back():
    from nanosim_b200.simulator import VERSION, bam_header
    m = bam_header()
    ms = bgzf_members(m)
    assert len(ms) == 1 and m[:16] == _zlib_member(b"")[:16]
    text, recs = read_bam(gzip.decompress(m))
    assert text == ("@HD\tVN:1.6\tSO:unknown\n@PG\tID:NanoSim\tPN:NanoSim\tVN:%s\n" % VERSION).encode() and recs == []
    assert b"CL:" not in text


def test_python_encoder_follows_the_specification():
    """The encoder the GPU tests compare against: fixed fields, packing of an odd-length read, the code table."""
    r = bam_record(b"rd", b"ACGTNacgtu=X", b"!" * 11 + b"I")
    assert struct.unpack_from("<i", r)[0] == 32 + 3 + 6 + 12 == len(r) - 4
    _, recs = read_bam(header_bytes() + r + bam_record(b"odd", b"ACG", None))
    a, b = recs
    assert a["codes"].tolist() == [1, 2, 4, 8, 15, 1, 2, 4, 8, 8, 0, 15] and a["qual"] == b"\0" * 11 + b"\x28"
    assert (a["ref_id"], a["pos"], a["mapq"], a["bin"], a["n_cigar"], a["flag"], a["next_ref_id"], a["next_pos"], a["tlen"]) == \
        (-1, -1, 255, 4680, 0, 4, -1, -1, 0)
    assert b["codes"].tolist() == [1, 2, 4] and b["pad"].tolist() == [0] and b["qual"] == b"\xff" * 3
    assert [_CODE[ord(c)] for c in SAM_CODES] == list(range(16)) and _CODE[ord("*")] == 15


def test_merge_rank_files_writes_the_header_and_one_eof(tmp_path):
    from nanosim_b200.simulator import bam_header, merge_rank_files
    out = os.path.join(str(tmp_path), "sim")
    parts = {}
    for kind in ("aligned", "unaligned"):
        for r in range(2):
            recs = [bam_record(b"%s_%d_%d" % (kind.encode(), r, i), b"ACGTA", None) for i in range(60)]
            parts[kind, r] = b"".join(_zlib_member(b"".join(recs[j:j + 20])) for j in range(0, 60, 20))
            with open(out + "_%s_reads%d.bam" % (kind, r), "wb") as f:
                f.write(parts[kind, r])
    for r in range(2):
        with open(out + "_error_profile%d" % r, "w") as f:
            f.write("r%d\t0\tmis\t1\tA\tC\n" % r)
    merge_rank_files(out, False, False, 2, bam=True)
    for kind in ("aligned", "unaligned"):
        path = out + "_%s_reads.bam" % kind
        assert open(path, "rb").read() == bam_header() + parts[kind, 0] + parts[kind, 1] + _eof()
        names = [r["name"] for r in read_bam(check_bgzf_file(path, quality=False))[1]]
        assert names == [b"%s_%d_%d" % (kind.encode(), r, i) for r in range(2) for i in range(60)]
        assert not os.path.exists(out + "_%s_reads0.bam" % kind)
    assert open(out + "_aligned_error_profile").read().endswith("r0\t0\tmis\t1\tA\tC\nr1\t0\tmis\t1\tA\tC\n")


def test_exports_name_the_new_entry_point():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    assert "ns_compress_bam" in _lib.EXPORTS and "ns_compress_bam(" in header
