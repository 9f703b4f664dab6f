"""--gzip_error_profile: the error profile formatted and compressed on the GPU (ns_compress_error_profile).

The device's rows must be the host formatter's bytes; every member must be valid BGZF; and every member must code the
repeated read names as the back-references bgzf_kernel.cuh defines, close to the optimal Huffman codes for that symbol
stream.  GPU tests run with ``pytest -m gpu``; the CLI-validation, naming and rank-merge tests at the end need no GPU."""
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
WINDOW = 32768
HEADER = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00"
ERR_HEADER = b"Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n"


def _eof():
    from nanosim_b200.simulator import BGZF_EOF
    return BGZF_EOF


def members(data):
    """Every member of a BGZF stream: (raw DEFLATE payload, CRC32, ISIZE), checking the header and BSIZE of each."""
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


def inflate_member(payload, crc, isize):
    d = zlib.decompressobj(-15)
    raw = d.decompress(payload) + d.flush()
    assert d.eof and not d.unused_data
    assert len(raw) == isize and zlib.crc32(raw) == crc
    return raw


def inflate(data):
    return b"".join(inflate_member(*m) for m in members(data))


# ------------------------------------------------------------------------- the matching rule of bgzf_kernel.cuh, restated
def _len_sym(n):
    """(symbol, extra bits) of a match length 3..258 (RFC 1951 §3.2.5)."""
    if n == 258:
        return 285, 0
    v = n - 3
    if v < 8:
        return 257 + v, 0
    e = v.bit_length() - 3
    return 261 + 4 * e + ((v >> e) & 3), e


def _dist_sym(d):
    v = d - 1
    if v < 4:
        return v, 0
    e = v.bit_length() - 2
    return 2 * e + 2 + ((v >> e) & 1), e


def _pieces(m):
    while m:
        n = m if m <= 258 else (m - 4 if m - 258 < 4 else 258)
        yield n
        m -= n


def block_symbols(text, b0, b1):
    """The symbol stream of the member for text[b0:b1): literal/length histogram (with end-of-block), distance histogram,
    extra bits.  A row starting at s whose previous row starts at p >= b0 is coded from s to min(s+f+1, b1) as
    back-references at distance s - p (f: bytes before the row's first TAB) when text[p:p+f+1] == text[s:s+f+1],
    s - p <= 32768 and that span has at least 4 bytes: pieces of 258, a short last one borrowing from the one before."""
    arr = np.frombuffer(text, dtype=np.uint8, count=b1 - b0, offset=b0)
    covered = np.zeros(b1 - b0, dtype=bool)
    ll, dist, extra = collections.Counter(), collections.Counter(), 0
    p = b0 if b0 == 0 or text[b0 - 1] == 10 else None
    for s in (b0 + np.flatnonzero(arr[:-1] == 10) + 1).tolist():
        prev, p = p, s
        if prev is None or s - prev > WINDOW:
            continue
        tab, nl = text.find(b"\t", s), text.find(b"\n", s)
        if tab < 0 or (0 <= nl < tab):
            continue
        f = tab - s
        if text[prev:prev + f + 1] != text[s:s + f + 1]:
            continue
        m = min(f + 1, b1 - s)
        if m < 4:
            continue
        covered[s - b0:s - b0 + m] = True
        for n in _pieces(m):
            sym, e = _len_sym(n)
            dsym, de = _dist_sym(s - prev)
            ll[sym] += 1
            dist[dsym] += 1
            extra += e + de
    for c, k in enumerate(np.bincount(arr[~covered], minlength=256).tolist()):
        if k:
            ll[c] += k
    ll[256] += 1
    return ll, dist, extra


def huffman_bits(counts):
    """Cost in bits of an optimal Huffman code for these symbol counts (one symbol alone costs a bit per use)."""
    heap = [c for c in counts if c]
    if len(heap) == 1:
        return heap[0]
    heapq.heapify(heap)
    bits = 0
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        bits += a + b
        heapq.heappush(heap, a + b)
    return bits


def check_profile_gz(path):
    """Structure and compression of a .gz error profile the simulator wrote; returns its decompressed bytes."""
    data = open(path, "rb").read()
    ms = members(data)
    assert data.endswith(_eof()) and ms[-1][2] == 0, path
    assert all(isize > 0 for _, _, isize in ms[:-1]), "%s: more than one end-of-file block" % path
    raws = [inflate_member(*m) for m in ms[:-1]]
    assert raws[0] == ERR_HEADER
    text = b"".join(raws)
    pos, payload_bytes, literal_bits = len(raws[0]), 0, 0
    for k, ((payload, _, isize), raw) in enumerate(zip(ms[1:-1], raws[1:])):
        assert 0 < isize <= BLOCK
        ll, dist, extra = block_symbols(text, pos, pos + isize)
        opt = (huffman_bits(ll.values()) + huffman_bits(dist.values()) + extra + 7) // 8
        assert opt <= len(payload) <= 1.01 * opt + 400, "%s member %d: %d bytes, optimal %d" % (path, k + 1, len(payload), opt)
        payload_bytes += len(payload)
        literal_bits += huffman_bits(list(collections.Counter(raw).values()) + [1])
        pos += isize
    assert payload_bytes < literal_bits / 8, "%s: %d bytes, literals only %d" % (path, payload_bytes, literal_bits // 8)
    return text


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def workdir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("errgz"))


def _guppy():
    return os.path.join(pc.DATA, pc.MODELS["guppy"])


def _meta_args(seed):
    from conftest import meta_fixture
    meta_fixture()                                          # writes genome_list_local.tsv
    M = os.path.join(GOLDEN, "meta")
    return ["metagenome", "-gl", os.path.join(M, "genome_list_local.tsv"), "-a", os.path.join(M, "abundance.tsv"), "-dl",
            os.path.join(M, "dna_type.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["even"]), "--fastq", "--chimeric", "--seed", str(seed)]


def _ir_args(seed, extra=()):
    D = os.path.join(GOLDEN, "ir")
    return ["transcriptome", "-rt", os.path.join(D, "transcripts.fa"), "-rg", os.path.join(D, "genome.fa"), "-e",
            os.path.join(D, "expression.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "--uracil",
            "--polya", os.path.join(D, "polya.txt"), "-b", "guppy", "--seed", str(seed),
            "--ir_markov_model", os.path.join(D, "IR_markov_model"), "--ir_gff3", os.path.join(D, "annotation.gff3")] + list(extra)


def _drna_hp_model(d):
    """The shipped dRNA model plus the dorado model's homopolymer table (it has none of its own), as one .npz."""
    from nanosim_b200.model import CompiledModel
    path = os.path.join(d, "drna_hp.npz")
    if not os.path.exists(path):
        cm = CompiledModel.load(os.path.join(pc.DATA, pc.MODELS["drna"]))
        hp = CompiledModel.load(os.path.join(pc.DATA, pc.MODELS["dorado"])).text["hp_lengths_model_parameters.tsv"]
        cm.text["hp_lengths_model_parameters.tsv"] = hp
        cm.save(path)
    return path


_MINI = os.path.join(GOLDEN, "mini_ref.fa")
_DEVICE_CONFIGS = {
    "guppy_fastq_chimeric_iupac": ["genome", "-rg", _MINI, "-c", _guppy(), "-n", "700", "--fastq", "--chimeric", "--seed", "41",
                                   "--batch_reads", "250"],
    "guppy_fasta": ["genome", "-rg", _MINI, "-c", _guppy(), "-n", "600", "--seed", "42", "--batch_reads", "250"],
    "circular": ["genome", "-rg", os.path.join(GOLDEN, "mini_circular.fa"), "-c", _guppy(), "-n", "600", "-dna_type", "circular",
                 "--seed", "43", "--batch_reads", "250"],
    "dorado_hp6_chimeric": ["genome", "-rg", _MINI, "-c", os.path.join(pc.DATA, pc.MODELS["dorado"]), "-n", "600", "--fastq", "-hp",
                            "-k", "6", "--chimeric", "--seed", "44", "--batch_reads", "250"],
    "metagenome_chimeric": None,
    "transcriptome_ir_uracil_hp6": None,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_DEVICE_CONFIGS))
def test_device_rows_equal_host_rows(name, workdir, monkeypatch):
    """Every aligned batch of a --gzip run (which still formats the profile on the host): the decompressed members of
    ns_compress_error_profile equal records.format_error_profile of the fetched batch."""
    from nanosim_b200 import _lib as L
    from nanosim_b200 import simulator
    from nanosim_b200.pipeline import BatchPipeline
    from nanosim_b200.records import format_error_profile
    args = _DEVICE_CONFIGS[name]
    if name == "metagenome_chimeric":
        args = _meta_args(45) + ["--batch_reads", "100"]
    elif name == "transcriptome_ir_uracil_hp6":
        args = _ir_args(46, ["-n", "1200", "-hp", "-k", "6", "--batch_reads", "400"])
        args[args.index("-c") + 1] = _drna_hp_model(workdir)
    seed = int(args[args.index("--seed") + 1])
    checked, mismatches = [], []
    orig = BatchPipeline._fetch_compressed

    def fetch(self, slot, job, info):
        b = orig(self, slot, job, info)
        if job[0] == L.NS_KIND_ALIGNED:
            eng = self.engines[slot]
            host = format_error_profile(b, b.names, eng.ref, seed=seed)
            n = eng.compress_error_profile(b.names)
            dev = eng.fetch_compressed_error_profile().tobytes()
            assert len(dev) == n
            got = inflate(dev)
            if got != host:
                k = next((i for i, (x, y) in enumerate(zip(got, host)) if x != y), min(len(got), len(host)))
                mismatches.append((job, len(got), len(host), got[max(0, k - 200):k + 100], host[max(0, k - 200):k + 100]))
            checked.append((len(host), b.pieces["kind"].copy(), b.pieces["ev_off"] != b.pieces["op_off"]))
        return b

    monkeypatch.setattr(BatchPipeline, "_fetch_compressed", fetch)
    simulator.main(args + ["-o", os.path.join(workdir, "dev_" + name), "-t", "4", "--gzip"])
    assert not mismatches, mismatches[0]
    assert len(checked) >= 2 * (2 if name == "metagenome_chimeric" else 1)
    assert sum(n for n, _, _ in checked) > 3 * BLOCK
    kinds = np.concatenate([k for _, k, _ in checked])
    rewritten = np.concatenate([r for _, _, r in checked])
    if "hp6" in name:
        assert rewritten.any()
    if name.startswith("transcriptome"):
        assert (kinds & L.NS_PIECE_REF_REV).any() and (kinds & L.NS_PIECE_CONT).any()


@pytest.mark.gpu
def test_device_rows_equal_python_rows_and_edge_cases():
    from nanosim_b200 import _lib as L
    from nanosim_b200.engine import NanoSimError
    from nanosim_b200.records import error_profile_rows, format_error_profile, name_table
    from nanosim_b200.reference_fasta import PackedReference
    ref = PackedReference.from_fasta(_MINI)
    eng, _, _ = pc.make_engine("guppy", ref, fastq=True, chimeric=True, seed=47)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 40)
    b = eng.fetch(want_ops=True)
    names = name_table(b, ref.names, 0)
    want = format_error_profile(b, names, ref, seed=47)
    assert want == "".join(error_profile_rows(b, names, ref, seed=47)).encode() and len(want) > 1000
    n = eng.compress_error_profile(names)
    dev = eng.fetch_compressed_error_profile().tobytes()
    assert inflate(dev) == want
    # repeated calls give the same bytes; records and profile in either order keep both results
    nr = eng.compress_records(names)
    recs = eng.fetch_compressed().tobytes()
    assert eng.compress_error_profile(names) == n and eng.fetch_compressed_error_profile().tobytes() == dev
    assert eng.fetch_compressed().tobytes() == recs and len(recs) == nr
    assert eng.compress_records(names) == nr and eng.fetch_compressed_error_profile().tobytes() == dev
    # too small a buffer
    with pytest.raises(NanoSimError, match="rc=-4"):
        eng.fetch_compressed_error_profile(np.empty(n - 1, dtype=np.uint8))
    # a one-read batch
    eng.simulate(L.NS_KIND_ALIGNED, 100, 1)
    b = eng.fetch(want_ops=True)
    names = name_table(b, ref.names, 100)
    want = format_error_profile(b, names, ref, seed=47)
    n = eng.compress_error_profile(names)
    assert inflate(eng.fetch_compressed_error_profile().tobytes()) == want and (n == 0) == (len(want) == 0)
    # unaligned reads have no profile
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 10)
    b = eng.fetch()
    with pytest.raises(NanoSimError, match="rc=-1"):
        eng.compress_error_profile(name_table(b, ref.names, 0))
    eng.close()


def _ecoli(tmp):
    ref = os.path.join(tmp, "ecoli5m.fa")
    if not os.path.exists(ref):
        synth.ecoli5m(ref)
    return ref


_CONFIGS = ["genome_fastq_chimeric", "genome_fasta", "dorado_fastq_hp6", "metagenome_chimeric", "transcriptome_ir_uracil"]
_RUNS = {}


def _run_config(name, tmp):
    """The configurations of test_bgzf_output.py, once with --gzip and once with --gzip --gzip_error_profile (same seed):
    the two output prefixes and the (reads, reads, error profile) file suffixes."""
    from nanosim_b200 import simulator
    if name in _RUNS:
        return _RUNS[name]
    ref = _ecoli(tmp)
    fq = ".fastq"
    if name == "genome_fastq_chimeric":
        args = ["genome", "-rg", ref, "-c", _guppy(), "-n", "2500", "--fastq", "--chimeric", "--seed", "21"]
    elif name == "genome_fasta":
        args = ["genome", "-rg", ref, "-c", _guppy(), "-n", "2500", "--seed", "22"]
        fq = ".fasta"
    elif name == "dorado_fastq_hp6":
        args = ["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["dorado"]), "-n", "2000", "--fastq", "-hp", "-k", "6",
                "--chimeric", "--seed", "23"]
    elif name == "metagenome_chimeric":
        args = _meta_args(24)
    else:
        args = _ir_args(25, ["-n", "1500", "--batch_reads", "600"])
        fq = ".fasta"
    plain, gz = os.path.join(tmp, name + "_gz"), os.path.join(tmp, name + "_gzerr")
    simulator.main(args + ["-o", plain, "-t", "4", "--gzip"])
    simulator.main(args + ["-o", gz, "-t", "4", "--gzip", "--gzip_error_profile"])
    prefixes = ["_sample0", "_sample1"] if name == "metagenome_chimeric" else [""]
    _RUNS[name] = (plain, gz, [(p + "_aligned_reads" + fq + ".gz", p + "_unaligned_reads" + fq + ".gz", p + "_aligned_error_profile")
                               for p in prefixes])
    return _RUNS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CONFIGS)
def test_cli_round_trip(name, workdir):
    plain, gz, files = _run_config(name, workdir)
    for al, un, err in files:
        for f in (al, un):
            assert open(plain + f, "rb").read() == open(gz + f, "rb").read(), f
        want = open(plain + err, "rb").read()
        assert len(want) > 1000 and not os.path.exists(gz + err)
        assert gzip.decompress(open(gz + err + ".gz", "rb").read()) == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["genome_fastq_chimeric", "dorado_fastq_hp6", "metagenome_chimeric", "transcriptome_ir_uracil"])
def test_members_are_valid_and_follow_the_rule(name, workdir):
    plain, gz, files = _run_config(name, workdir)
    for _, _, err in files:
        text = check_profile_gz(gz + err + ".gz")
        assert text == open(plain + err, "rb").read()
    if name == "genome_fastq_chimeric":
        assert len(text) > 4 * BLOCK


@pytest.mark.gpu
def test_output_is_independent_of_batching(tmp_path):
    from nanosim_b200 import simulator
    ref = _ecoli(str(tmp_path))
    outs = []
    for batch in ("700", "5000"):
        out = os.path.join(str(tmp_path), "b" + batch)
        simulator.main(["genome", "-rg", ref, "-c", _guppy(), "-n", "4000", "--fastq", "--seed", "34", "--batch_reads", batch, "-t", "3",
                        "--gzip", "--gzip_error_profile", "-o", out])
        outs.append(out)
    a, b = (gzip.decompress(open(o + "_aligned_error_profile.gz", "rb").read()) for o in outs)
    assert a == b and a.startswith(ERR_HEADER) and len(a) > 10 * BLOCK


@pytest.mark.gpu
def test_pipeline_fetches_neither_bases_nor_ops(tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    from nanosim_b200.engine import Engine
    calls = []
    orig = Engine.fetch_into

    def fetch_into(self, seq_ptr, qual_ptr, reads_ptr, pieces_ptr=None, ops_ptr=None):
        calls.append((seq_ptr, qual_ptr, ops_ptr))
        return orig(self, seq_ptr, qual_ptr, reads_ptr, pieces_ptr, ops_ptr)

    monkeypatch.setattr(Engine, "fetch_into", fetch_into)
    out = os.path.join(str(tmp_path), "s")
    simulator.main(["genome", "-rg", _MINI, "-c", _guppy(), "-n", "600", "--fastq", "--seed", "48", "--batch_reads", "200",
                    "--gzip", "--gzip_error_profile", "-o", out])
    assert len(calls) >= 3 and all(c == (None, None, None) for c in calls)
    assert gzip.decompress(open(out + "_aligned_error_profile.gz", "rb").read()).count(b"\n") > 100


@pytest.mark.gpu
@pytest.mark.multigpu
def test_two_ranks_equal_one_rank_plain(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = _ecoli(str(tmp_path))
    args = ["genome", "-rg", ref, "-c", _guppy(), "-n", "4000", "--fastq", "--seed", "35", "--batch_reads", "700", "-t", "4"]
    one, two = os.path.join(str(tmp_path), "one"), os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29744", "-m", "nanosim_b200.simulator"] + args + ["-o", two, "--gzip", "--gzip_error_profile"],
                   check=True, env=env, cwd=ROOT)
    assert check_profile_gz(two + "_aligned_error_profile.gz") == open(one + "_aligned_error_profile", "rb").read()
    assert not os.path.exists(two + "_error_profile1.gz")


# ---------------------------------------------------------------------------------------------------------------- CPU
_ARGV = {"genome": ["genome", "-rg", "x.fa"], "metagenome": ["metagenome", "-gl", "gl.tsv", "-a", "ab.tsv"],
         "transcriptome": ["transcriptome", "-rt", "t.fa", "-e", "e.tsv", "--no_model_ir"]}


@pytest.mark.parametrize("mode", list(_ARGV))
def test_flag_needs_gzip(mode, tmp_path, capsys):
    from nanosim_b200 import simulator
    with pytest.raises(SystemExit) as e:
        simulator.main(_ARGV[mode] + ["-o", os.path.join(str(tmp_path), "sim"), "--gzip_error_profile"])
    assert e.value.code == 1
    assert "--gzip_error_profile needs --gzip" in capsys.readouterr().err
    assert os.listdir(str(tmp_path)) == []


class _NoGpuEngine:
    def configure(self, **kw):
        pass

    def set_abundance(self, *a):
        pass


class _EmptyPipeline:
    """Stands in for BatchPipeline when a run has no reads: nothing to simulate, the output files are still written."""

    kw = None

    def __init__(self, *a, **kw):
        self.want_ops, self.compress, self.compress_profile = kw.get("want_ops"), None, kw.get("compress_profile")
        _EmptyPipeline.kw = kw

    def run(self, jobs, consume=None, **kw):
        assert list(jobs) == []
        return []

    def close(self):
        pass


def _empty_profile(*a, **kw):
    from nanosim_b200 import simulator
    assert kw.get("ref_on_host") is False
    prof = simulator.Profile()
    prof.engine, prof.ir, prof.n_trx, prof.seed, prof.max_chrom = _NoGpuEngine(), None, 0, 0, 1000
    prof.tables = types.SimpleNamespace(abun_inflation=1.0, split_counts=lambda n, per: (0, 0))
    prof.ref = types.SimpleNamespace(names=["c"], lengths=np.array([1000]), chrom_species=np.array([0]), species=["s"],
                                     max_chrom_per_species={"s": 1000}, max_chrom=1000)
    prof.samples, prof.counts = [[100.0]], [(0, 0)]
    return prof


@pytest.mark.parametrize("mode", list(_ARGV))
def test_flag_names_the_outputs(mode, tmp_path, monkeypatch):
    from nanosim_b200 import simulator
    monkeypatch.setattr(simulator, "read_profile", _empty_profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(_ARGV[mode] + ["-o", out, "--gzip", "--gzip_error_profile", "--fastq"])
    assert _EmptyPipeline.kw["compress_profile"] and not _EmptyPipeline.kw["want_ops"]
    prefix = out + ("_sample0" if mode == "metagenome" else "")
    data = open(prefix + "_aligned_error_profile.gz", "rb").read()
    assert gzip.decompress(data) == ERR_HEADER and data.endswith(_eof()) and len(members(data)) == 2
    assert not os.path.exists(prefix + "_aligned_error_profile")
    assert open(prefix + "_aligned_reads.fastq.gz", "rb").read() == _eof()


def test_no_error_profile_keeps_the_plain_file(tmp_path, monkeypatch):
    """--no_error_profile: nothing to compress, the plain header-only file is written as without the flag."""
    from nanosim_b200 import simulator
    monkeypatch.setattr(simulator, "read_profile", _empty_profile)
    monkeypatch.setattr(simulator, "BatchPipeline", _EmptyPipeline)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(_ARGV["genome"] + ["-o", out, "--gzip", "--gzip_error_profile", "--no_error_profile"])
    assert not _EmptyPipeline.kw["compress_profile"]
    assert open(out + "_aligned_error_profile", "rb").read() == ERR_HEADER
    assert not os.path.exists(out + "_aligned_error_profile.gz")


def _zlib_member(text):
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(text) + c.flush()
    return HEADER + struct.pack("<H", 18 + len(payload) + 8 - 1) + payload + struct.pack("<II", zlib.crc32(text), len(text))


def test_merge_rank_files_writes_header_members_and_one_eof(tmp_path):
    from nanosim_b200.simulator import bgzf_member, merge_rank_files
    out = os.path.join(str(tmp_path), "sim")
    parts, texts = [], []
    for r in range(2):
        t = [b"".join(b"r%d_%d\t%d\tmis\t1\tA\tC\n" % (r, j, i) for i in range(40)) for j in range(3)]
        texts.append(b"".join(t))
        parts.append(b"".join(_zlib_member(x) for x in t))
        with open(out + "_error_profile%d.gz" % r, "wb") as f:
            f.write(parts[r])
        for kind in ("aligned", "unaligned"):
            with open(out + "_%s_reads%d.fasta.gz" % (kind, r), "wb") as f:
                f.write(_zlib_member(b">x\nACGT\n"))
    merge_rank_files(out, False, False, 2, gzip=True, gzip_error_profile=True)
    data = open(out + "_aligned_error_profile.gz", "rb").read()
    assert data == bgzf_member(ERR_HEADER) + parts[0] + parts[1] + _eof()
    assert inflate(data) == ERR_HEADER + texts[0] + texts[1] and gzip.decompress(data) == ERR_HEADER + texts[0] + texts[1]
    assert not os.path.exists(out + "_error_profile0.gz") and not os.path.exists(out + "_aligned_error_profile")


def test_header_member_is_bgzf():
    from nanosim_b200.simulator import bgzf_member
    m = bgzf_member(ERR_HEADER)
    assert len(ERR_HEADER) == 59 and [inflate_member(*x) for x in members(m)] == [ERR_HEADER]


def test_exports_name_the_new_entry_points():
    from nanosim_b200 import _lib
    header = open(os.path.join(ROOT, "include", "nanosim_b200.h")).read()
    for name in ("ns_compress_error_profile", "ns_fetch_compressed_error_profile"):
        assert name in _lib.EXPORTS and (name + "(") in header
