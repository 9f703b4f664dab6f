"""--gzip: the reads files as BGZF, compressed on the GPU (ns_compress_records).

Decompressed, every .gz file must be the plain file of the same run byte for byte; each member must be a valid BGZF
member that inflates on its own; and each member's single Huffman code must be close to the optimal one for its bytes.
GPU tests run with ``pytest -m gpu``; the CLI and rank-merge tests at the end need no GPU."""
import collections
import gzip
import heapq
import os
import struct
import subprocess
import sys
import types
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

import parity_checks as pc
import synth

BLOCK = 56 * 1024          # uncompressed bytes per member (nanosim_b200/csrc/bgzf_kernel.cuh: BGZF_BLOCK)
HEADER = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00"


def _eof():
    from nanosim_b200.simulator import BGZF_EOF
    return BGZF_EOF


def bgzf_members(data):
    """Every member of a BGZF file: (raw DEFLATE payload, CRC32, ISIZE), checking the header and BSIZE of each."""
    out, pos = [], 0
    while pos < len(data):
        h = data[pos:pos + 18]
        assert h[:16] == HEADER, "member at %d: bad header %r" % (pos, h)
        size = struct.unpack("<H", h[16:18])[0] + 1
        assert size <= 65536 and pos + size <= len(data), "member at %d: BSIZE + 1 = %d" % (pos, size)
        crc, isize = struct.unpack("<II", data[pos + size - 8:pos + size])
        out.append((data[pos + 18:pos + size - 8], crc, isize))
        pos += size
    return out


def huffman_bits(raw):
    """Cost in bits of an optimal Huffman code over the bytes' histogram plus the end-of-block symbol DEFLATE needs."""
    heap = list(collections.Counter(raw).values()) + [1]
    heapq.heapify(heap)
    bits = 0
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        bits += a + b
        heapq.heappush(heap, a + b)
    return bits


def check_bgzf_file(path, quality=True):
    """Structure (and compression quality) of a file the simulator wrote; returns its decompressed bytes."""
    data = open(path, "rb").read()
    ms = bgzf_members(data)
    assert data.endswith(_eof()) and ms[-1][2] == 0, path
    assert all(isize > 0 for _, _, isize in ms[:-1]), "%s: more than one end-of-file block" % path
    text = []
    for k, (payload, crc, isize) in enumerate(ms[:-1]):
        assert isize <= BLOCK
        d = zlib.decompressobj(-15)
        raw = d.decompress(payload) + d.flush()
        assert d.eof and not d.unused_data
        assert len(raw) == isize and zlib.crc32(raw) == crc, "%s member %d" % (path, k)
        if quality:
            opt = (huffman_bits(raw) + 7) // 8
            assert len(payload) <= 1.01 * opt + 300, "%s member %d: %d bytes, optimal Huffman %d" % (path, k, len(payload), opt)
        text.append(raw)
    return b"".join(text)


# ---------------------------------------------------------------------------------------------------------------- GPU
_CONFIGS = ["genome_fastq_chimeric", "genome_fasta", "dorado_fastq_hp6", "metagenome_chimeric", "transcriptome_ir_uracil"]
_RUNS = {}


def _run_config(name, tmp):
    """Runs the configuration once without and once with --gzip (same seed): returns the two output prefixes and the
    reads / error-profile suffixes to compare."""
    from nanosim_b200 import simulator
    from conftest import meta_fixture
    if name in _RUNS:
        return _RUNS[name]
    ref = os.path.join(tmp, "ecoli5m.fa")
    if not os.path.exists(ref):
        synth.ecoli5m(ref)
    fq = ".fastq"
    if name == "genome_fastq_chimeric":
        args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "2500", "--fastq", "--chimeric", "--seed", "21"]
    elif name == "genome_fasta":
        args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "2500", "--seed", "22"]
        fq = ".fasta"
    elif name == "dorado_fastq_hp6":
        args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["dorado"]), "-n", "2000", "--fastq", "-hp", "-k", "6",
                "--chimeric", "--seed", "23"]
    elif name == "metagenome_chimeric":
        meta_fixture()                                          # writes genome_list_local.tsv
        M = os.path.join(GOLDEN, "meta")
        args = ["metagenome", "-gl", os.path.join(M, "genome_list_local.tsv"), "-a", os.path.join(M, "abundance.tsv"), "-dl",
                os.path.join(M, "dna_type.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["even"]), "--fastq", "--chimeric", "--seed", "24"]
    else:
        D = os.path.join(GOLDEN, "ir")
        args = ["transcriptome", "-rt", os.path.join(D, "transcripts.fa"), "-rg", os.path.join(D, "genome.fa"), "-e",
                os.path.join(D, "expression.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", "1500", "--uracil",
                "--polya", os.path.join(D, "polya.txt"), "-b", "guppy", "--seed", "25", "--batch_reads", "600",
                "--ir_markov_model", os.path.join(D, "IR_markov_model"), "--ir_gff3", os.path.join(D, "annotation.gff3")]
        fq = ".fasta"
    plain, gz = os.path.join(tmp, name + "_plain"), os.path.join(tmp, name + "_gz")
    simulator.main(args + ["-o", plain, "-t", "4"])
    simulator.main(args + ["-o", gz, "-t", "4", "--gzip"])
    prefixes = ["_sample0", "_sample1"] if name == "metagenome_chimeric" else [""]
    _RUNS[name] = (plain, gz, [(p + "_aligned_reads" + fq, p + "_unaligned_reads" + fq, p + "_aligned_error_profile") for p in prefixes])
    return _RUNS[name]


@pytest.fixture(scope="module")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("bgzf"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_gzip_output_decompresses_to_the_plain_output(name, workdir):
    plain, gz, files = _run_config(name, workdir)
    for al, un, err in files:
        for f in (al, un):
            want = open(plain + f, "rb").read()
            assert len(want) > 1000 and not os.path.exists(gz + f)
            assert gzip.decompress(open(gz + f + ".gz", "rb").read()) == want, f
        assert open(plain + err, "rb").read() == open(gz + err, "rb").read(), err
    if name == "transcriptome_ir_uracil":
        text = open(plain + files[0][0], "rb").read()
        seqs = text.split(b"\n")[1::2]
        assert b"_RetainedIntron_" in text and all(b"T" not in x for x in seqs) and any(b"U" in x for x in seqs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_bgzf_members_are_valid_and_near_optimal(name, workdir):
    plain, gz, files = _run_config(name, workdir)
    for al, un, _ in files:
        for f in (al, un):
            assert check_bgzf_file(gz + f + ".gz") == open(plain + f, "rb").read()


@pytest.fixture(scope="module")
def ecoli():
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_records(synth.ecoli5m())


def _compress_batch(eng, ref, kind, n, first=0):
    """Simulates one batch, formats it on the host and compresses it on the device: (plain text, members)."""
    from nanosim_b200.records import format_records, name_table
    eng.simulate(kind, first, n)
    b = eng.fetch()
    names = name_table(b, ref.names, first)
    plain = format_records(b, names, eng.fastq)
    nz = eng.compress_records(names)
    members = eng.fetch_compressed().tobytes()
    assert len(members) == nz
    return plain, members, names


@pytest.mark.gpu
def test_one_read_batch_and_fetch_capacity(ecoli):
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import NanoSimError
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=True, seed=31)
    plain, members, names = _compress_batch(eng, ecoli, L.NS_KIND_ALIGNED, 1)
    assert len(plain) < BLOCK and len(bgzf_members(members)) == 1
    assert gzip.decompress(members + _eof()) == plain
    assert eng.compress_records(names) == len(members) and eng.fetch_compressed().tobytes() == members   # deterministic
    with pytest.raises(NanoSimError, match="rc=-4"):
        eng.fetch_compressed(np.empty(len(members) - 1, dtype=np.uint8))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fastq", [False, True])
def test_reads_longer_than_several_blocks(ecoli, fastq, tmp_path):
    from nanosim_b200 import _lib as L
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=fastq, seed=32)
    eng.configure(fastq=fastq, min_len=200000, max_len=ecoli.max_chrom, median_len=300000, sd_len=0.1)
    plain, members, _ = _compress_batch(eng, ecoli, L.NS_KIND_ALIGNED, 5)
    assert eng.info.total_bases / 5 > 3 * BLOCK
    path = os.path.join(str(tmp_path), "long.gz")
    with open(path, "wb") as f:
        f.write(members + _eof())
    assert check_bgzf_file(path) == plain
    eng.close()


@pytest.mark.gpu
def test_names_with_bytes_above_0x7f(tmp_path):
    """Reference headers with UTF-8 letters put bytes >= 0x80 into the read names."""
    from nanosim_b200 import simulator
    ref = os.path.join(str(tmp_path), "utf8.fa")
    with open(os.path.join(GOLDEN, "mini_ref.fa"), "rb") as f, open(ref, "wb") as o:
        k = 0
        for line in f:
            if line.startswith(b">"):
                line = (">chr_%d_éß中 desc\n" % k).encode()
                k += 1
            o.write(line)
    args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "1500", "--fastq", "--seed", "33"]
    plain, gz = os.path.join(str(tmp_path), "p"), os.path.join(str(tmp_path), "g")
    simulator.main(args + ["-o", plain])
    simulator.main(args + ["-o", gz, "--gzip"])
    for f in ("_aligned_reads.fastq", "_unaligned_reads.fastq"):
        want = open(plain + f, "rb").read()
        assert "éß中".encode() in want
        assert check_bgzf_file(gz + f + ".gz") == want


@pytest.mark.gpu
def test_decompressed_output_is_independent_of_batching(tmp_path):
    from nanosim_b200 import simulator
    ref = os.path.join(str(tmp_path), "ecoli5m.fa")
    synth.ecoli5m(ref)
    outs = []
    for batch in ("700", "5000"):
        out = os.path.join(str(tmp_path), "b" + batch)
        simulator.main(["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "4000", "--fastq", "--seed", "34",
                        "--batch_reads", batch, "-t", "3", "--gzip", "-o", out])
        outs.append(out)
    for f in ("_aligned_reads.fastq.gz", "_unaligned_reads.fastq.gz"):
        a, b = (gzip.decompress(open(o + f, "rb").read()) for o in outs)
        assert a == b and len(a) > 1000, f


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_gzip_equal_one_rank_plain(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = os.path.join(str(tmp_path), "ecoli5m.fa")
    synth.ecoli5m(ref)
    args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "4000", "--fastq", "--seed", "35",
            "--batch_reads", "700", "-t", "4"]
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29743", "-m", "nanosim_b200.simulator"] + args + ["-o", two, "--gzip"], check=True, env=env, cwd=ROOT)
    for f in ("_aligned_reads.fastq", "_unaligned_reads.fastq"):
        assert check_bgzf_file(two + f + ".gz") == open(one + f, "rb").read(), f
    assert open(one + "_aligned_error_profile", "rb").read() == open(two + "_aligned_error_profile", "rb").read()
    assert not os.path.exists(two + "_aligned_reads1.fastq.gz")


# ---------------------------------------------------------------------------------------------------------------- CPU
class _NoGpuEngine:
    def configure(self, **kw):
        pass

    def set_abundance(self, *a):
        pass


class _EmptyPipeline:
    """Stands in for BatchPipeline when a run has no reads: nothing to simulate, the output files are still written."""

    def __init__(self, *a, **kw):
        self.want_ops, self.compress = kw.get("want_ops"), None

    def run(self, jobs, consume=None, **kw):
        assert list(jobs) == []
        return []

    def close(self):
        pass


def _empty_profile(*a, **kw):
    from nanosim_b200 import simulator
    prof = simulator.Profile()
    prof.engine, prof.ir, prof.n_trx, prof.seed, prof.max_chrom = _NoGpuEngine(), None, 0, 0, 1000
    prof.tables = types.SimpleNamespace(abun_inflation=1.0, split_counts=lambda n, per: (0, 0))
    prof.ref = types.SimpleNamespace(names=["c"], lengths=np.array([1000]), chrom_species=np.array([0]), species=["s"],
                                     max_chrom_per_species={"s": 1000}, max_chrom=1000)
    prof.samples, prof.counts = [[100.0]], [(0, 0)]
    return prof


@pytest.mark.parametrize("mode", ["genome", "metagenome", "transcriptome"])
@pytest.mark.parametrize("fastq", [False, True])
def test_gzip_flag_names_the_outputs(mode, fastq, tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    monkeypatch.setattr(simulator, "read_profile", _empty_profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    argv = {"genome": ["genome", "-rg", "x.fa"], "metagenome": ["metagenome", "-gl", "gl.tsv", "-a", "ab.tsv"],
            "transcriptome": ["transcriptome", "-rt", "t.fa", "-e", "e.tsv", "--no_model_ir"]}[mode]
    simulator.main(argv + ["-o", out, "--gzip"] + (["--fastq"] if fastq else []))
    prefix = out + ("_sample0" if mode == "metagenome" else "")
    ext = ".fastq" if fastq else ".fasta"
    for f in ("_aligned_reads", "_unaligned_reads"):
        assert open(prefix + f + ext + ".gz", "rb").read() == _eof()
        assert gzip.decompress(_eof()) == b""
        assert not os.path.exists(prefix + f + ext)
    assert open(prefix + "_aligned_error_profile").read().startswith("Seq_name\t")


def _zlib_member(text):
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(text) + c.flush()
    return HEADER + struct.pack("<H", 18 + len(payload) + 8 - 1) + payload + struct.pack("<II", zlib.crc32(text), len(text))


def test_merge_rank_files_appends_one_eof_block(tmp_path):
    from nanosim_b200.simulator import merge_rank_files
    out = os.path.join(str(tmp_path), "sim")
    parts, texts = {}, {}
    for kind in ("aligned", "unaligned"):
        for r in range(2):
            t = [b"".join(b">%s_%d_%d\nACGT\n" % (kind.encode(), r, i) for i in range(j * 50, j * 50 + 50)) for j in range(3)]
            texts[kind, r] = b"".join(t)
            parts[kind, r] = b"".join(_zlib_member(x) for x in t)
            with open(out + "_%s_reads%d.fasta.gz" % (kind, r), "wb") as f:
                f.write(parts[kind, r])
    for r in range(2):
        with open(out + "_error_profile%d" % r, "w") as f:
            f.write("r%d\t0\tmis\t1\tA\tC\n" % r)
    merge_rank_files(out, False, False, 2, gzip=True)
    for kind in ("aligned", "unaligned"):
        path = out + "_%s_reads.fasta.gz" % kind
        assert open(path, "rb").read() == parts[kind, 0] + parts[kind, 1] + _eof()
        assert check_bgzf_file(path, quality=False) == texts[kind, 0] + texts[kind, 1]
        assert gzip.decompress(open(path, "rb").read()) == texts[kind, 0] + texts[kind, 1]
        assert not os.path.exists(out + "_%s_reads0.fasta.gz" % kind)
    assert open(out + "_aligned_error_profile").read() == "Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\nr0\t0\tmis\t1\tA\tC\nr1\t0\tmis\t1\tA\tC\n"
