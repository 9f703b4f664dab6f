"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Everything goes through the C ABI.

 * bit-exact: every edit script re-applied on the host reproduces the device's bases (mutate_read semantics);
   same seed -> same bytes; results independent of the batch split;
 * statistical, vs the oracle run here on a few hundred reads;
 * statistical, vs the committed histograms of the UNMODIFIED reference (tests/golden/ref_stats_*.json, 1M reads):
   per-base mis/ins/del counts within +-0.1 % (north_star), length / event histograms by chi-square.
"""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN

import parity_checks as pc
import run_stats as rs
import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from nanosim_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def mini_ref():
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_fasta(os.path.join(GOLDEN, "mini_ref.fa"))


@pytest.fixture(scope="module")
def ecoli():
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_records(synth.ecoli5m())


CONFIGS = [
    ("guppy", dict(fastq=True)),
    ("guppy", dict(fastq=False)),
    ("dorado", dict(fastq=True, chimeric=True)),
    ("guppy", dict(fastq=True, perfect=True)),
]


@pytest.mark.parametrize("model,kw", CONFIGS)
def test_edit_scripts_bit_exact_mini_ref(model, kw, mini_ref, L):
    """Reference with lower case, IUPAC codes and three chromosomes (reads never span chromosomes)."""
    eng, cm, t = pc.make_engine(model, mini_ref, seed=3, **kw)
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, 1500)
    b = eng.fetch(want_ops=True)
    assert info.n_reads == 1500 and int(b.reads["seq_len"].astype(np.int64).sum()) == info.total_bases
    assert pc.check_edit_scripts(b, mini_ref, kw.get("fastq", False)) > 0
    lens = b.reads["seq_len"]
    assert lens.min() >= 50 and lens.max() <= mini_ref.max_chrom
    if kw.get("perfect"):
        assert (b.reads["head"] == 0).all() and (b.reads["tail"] == 0).all()
        assert ((b.ops >> 28) == 0).all()
    eng.close()


@pytest.mark.parametrize("model,fastq", [("guppy", True), ("guppy", False), ("dorado", True)])
def test_unaligned_fast_path_equals_scripted_path(model, fastq, mini_ref, L):
    """The warp-per-read unaligned kernel evaluates unaligned_error_list 32 draws at a time; the scripted path runs
    it sequentially and keeps edit scripts.  Same seed => same lengths, rejections, strands and positions, and the
    fast path's bytes must equal the scripted path's and satisfy both paths' edit scripts bit-exactly."""
    a, _, _ = pc.make_engine(model, mini_ref, fastq=fastq, seed=21, unaligned_scripts=True)
    a.simulate(L.NS_KIND_UNALIGNED, 100, 1500)
    bs = a.fetch(want_ops=True)
    assert pc.check_edit_scripts(bs, mini_ref, fastq) > 0
    a.close()
    b, _, _ = pc.make_engine(model, mini_ref, fastq=fastq, seed=21)
    info = b.simulate(L.NS_KIND_UNALIGNED, 100, 1500)
    bf = b.fetch(want_ops=True)
    b.close()
    assert info.n_ops > 0 and bf.reads["seq_len"].min() >= 50
    assert pc.check_fast_unaligned(bf, bs, mini_ref, fastq) > 0
    assert bf.reads["attempts"].max() > 0


def _reads_bytes(b, fastq):
    out = []
    for r in b.reads:
        a, n = int(r["seq_off"]), int(r["seq_len"])
        out.append((b.seq[a:a + n].tobytes(), b.qual[a:a + n].tobytes() if fastq else b""))
    return out


@pytest.mark.parametrize("model,kw", [("guppy", dict(fastq=True)), ("guppy", dict(fastq=False)),
                                      ("dorado", dict(fastq=True, chimeric=True)), ("dorado", dict(fastq=True, chimeric=True, kmer_bias=6))])
def test_emit_fast_route_equals_exact_route(model, kw, ecoli, mini_ref, L):
    """The emit kernel reads plain-ACGT stretches from the 2-bit copy of the reference, 16 bases per entry (fast route), and
    everything else byte by byte (exact route).  Same seed => same bytes on either route: on a pure-ACGT reference every
    piece is fast, NS_FLAG_EMIT_EXACT forces the other route; on the IUPAC / lower-case mini reference the routes mix."""
    fastq = kw.get("fastq", False)
    for ref in (ecoli, mini_ref):
        got = {}
        for exact in (False, True):
            eng, _, _ = pc.make_engine(model, ref, seed=314, emit_exact=exact, **kw)
            eng.simulate(L.NS_KIND_ALIGNED, 11, 4000)
            b = eng.fetch(want_ops=True)
            if not exact:
                assert pc.check_edit_scripts(b, ref, fastq, max_reads=300) > 0
            rows = _reads_bytes(b, fastq)
            eng.simulate(L.NS_KIND_UNALIGNED, 5, 800)
            rows += _reads_bytes(eng.fetch(), fastq)
            eng.close()
            got[exact] = rows
        n_diff = sum(x != y for x, y in zip(got[False], got[True]))
        assert len(got[False]) == len(got[True]) == 4800 and n_diff == 0, "%d reads differ between the routes" % n_diff


@pytest.mark.parametrize("model,kw", [("guppy", dict(fastq=True)), ("dorado", dict(fastq=False, chimeric=True)),
                                      ("dorado", dict(fastq=True, chimeric=True, kmer_bias=6))])
def test_emit_split_pieces_equal_whole_pieces(model, kw, ecoli, mini_ref, L):
    """Pieces longer than 16 kb are emitted as several work items, each resuming the script walk from a checkpoint
    (emit_kernel.cuh:split_kernel); NS_FLAG_EMIT_WHOLE emits every piece in one go.  Same bytes either way, on both routes
    (pure-ACGT reference: fast; IUPAC / lower-case mini reference: mixed), forward and reverse reads, aligned and unaligned."""
    fastq = kw.get("fastq", False)
    for ref, exact in ((ecoli, False), (ecoli, True), (mini_ref, False)):
        got, n_long = {}, 0
        for whole in (False, True):
            eng, _, _ = pc.make_engine(model, ref, seed=2718, emit_whole=whole, emit_exact=exact, **kw)
            eng.simulate(L.NS_KIND_ALIGNED, 3, 3000)
            b = eng.fetch(want_ops=True)
            if not whole:
                assert pc.check_edit_scripts(b, ref, fastq, max_reads=200) > 0
                n_long = int((b.pieces["out_len"] > 40000).sum())
            rows = _reads_bytes(b, fastq)
            eng.simulate(L.NS_KIND_UNALIGNED, 9, 1500)
            rows += _reads_bytes(eng.fetch(), fastq)
            eng.close()
            got[whole] = rows
        if ref is ecoli:
            assert n_long > 0, "no piece long enough to be split three ways: the test does not test anything"
        n_diff = sum(x != y for x, y in zip(got[False], got[True]))
        assert len(got[False]) == len(got[True]) == 4500 and n_diff == 0, "%d reads differ between split and whole emission" % n_diff


def test_unaligned_event_scripts_vs_oracle(ecoli, L, tmp_path):
    """unaligned_error_list (simulator.py:1784-1830: 0.4/0.3/0.15/0.15 step mix, insertions merged at pos+0.1) and what
    mutate_read makes of its e_dict (:1957-1995) against the pinned oracle: the device's scripted unaligned path on 2500
    reads vs oracle.unaligned_error_list on the same drawn lengths.  The oracle's e_dict is turned into per-base
    provenance by the splice arithmetic of mutate_read on tags, and that is checked against oracle.mutate_read on a
    random string for every read, so the comparison stands on the oracle alone."""
    import random
    import nanosim_oracle as no
    from conftest import oracle_model
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=False, seed=57, unaligned_scripts=True, max_len=30000)
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 2500)
    b = eng.fetch(want_ops=True)
    eng.close()
    assert pc.check_edit_scripts(b, ecoli, False) > 0
    dev_ops = [pc.device_piece_ops(b, pcs) for pcs in b.pieces]
    s_dev = pc.script_stats(dev_ops, canonical=True)       # INS/DEL that touch have no order
    m = oracle_model(cm, tmp_path, fastq=False)
    random.seed(99)
    np.random.seed(99)
    or_ops, d_len_dev, d_len_or = [], [], []
    alphabet = "ACGT"
    for pcs in b.pieces:
        m_ref = int(pcs["ref_req"])
        l_new, middle_ref, e_dict, e_count = no.unaligned_error_list(m_ref, m)
        tags = pc.apply_edict_to_tags(e_dict, middle_ref)
        read = "".join(random.choice(alphabet) for _ in range(middle_ref))
        mutated, _ = no.mutate_read(read, "x", None, dict(e_dict), e_count, False, False, m)
        assert len(mutated) == len(tags)
        for ch, tg in zip(mutated, tags):                      # the tag interpreter agrees with the oracle's strings
            if isinstance(tg, int):
                assert ch == read[tg]
            elif isinstance(tg, tuple) and isinstance(tg[1], int):
                assert ch != read[tg[1]]
        or_ops.append(pc.tags_to_ops(tags, middle_ref))
        d_len_or.append((len(tags) - m_ref, middle_ref - m_ref))
        d_len_dev.append((int(pcs["out_len"]) - m_ref, int(pcs["ref_len"]) - m_ref))
    s_or = pc.script_stats(or_ops, canonical=True)
    rd, ro = pc.rates(s_dev), pc.rates(s_or)
    print("unaligned per-reference-base event bases device", rd, "oracle", ro)
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.02, p_min=1e-5, label="unaligned-scripts",
                             keys=["match_run", "first_match", "events_per_read"])
    for k in ("mis", "ins", "del"):
        a, o = s_dev["events"][k] / s_dev["ref_bases"], s_or["events"][k] / s_or["ref_bases"]
        if abs(a / o - 1) > 0.02:
            fails.append("unaligned %s events per reference base %.5f vs %.5f" % (k, a, o))
    # read length minus drawn length, and the overshoot of the last step (:1826-1828)
    d_len_dev, d_len_or = np.asarray(d_len_dev, dtype=np.float64), np.asarray(d_len_or, dtype=np.float64)
    scale = np.sqrt(np.maximum(b.pieces["ref_req"].astype(np.float64), 1.0))
    edges = np.linspace(-6, 6, 41)
    st, dof, p = pc.chi2_two_sample(np.histogram(d_len_dev[:, 0] / scale, edges)[0], np.histogram(d_len_or[:, 0] / scale, edges)[0])
    print("normalised length change chi2 %.1f dof %d p %.3g; mean %.2f vs %.2f" % (st, dof, p, d_len_dev[:, 0].mean(), d_len_or[:, 0].mean()))
    if p < 1e-5:
        fails.append("unaligned length change: chi2 %.1f dof %d p %.3g" % (st, dof, p))
    st, dof, p = pc.chi2_two_sample(np.bincount(d_len_dev[:, 1].astype(np.int64), minlength=12)[:12],
                                    np.bincount(d_len_or[:, 1].astype(np.int64), minlength=12)[:12], min_count=10)
    print("overshoot of the last step chi2 %.1f dof %d p %.3g" % (st, dof, p))
    if p < 1e-5:
        fails.append("unaligned overshoot: chi2 %.1f dof %d p %.3g" % (st, dof, p))
    assert not fails, "\n".join(fails)


def test_circular_reference_wraps(L):
    from nanosim_b200.reference_fasta import PackedReference
    ref = PackedReference.from_fasta(os.path.join(GOLDEN, "mini_circular.fa"))
    eng, cm, t = pc.make_engine("dorado", ref, fastq=True, seed=5, circular=True, max_len=4000)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 2000)
    b = eng.fetch(want_ops=True)
    assert pc.check_edit_scripts(b, ref, True) > 0
    seg = b.pieces[b.pieces["kind"] == L.NS_PIECE_SEGMENT]
    wrapped = (seg["pos"].astype(np.int64) + seg["ref_len"].astype(np.int64)) > ref.genome_len
    assert wrapped.any(), "no read wrapped around the circular chromosome"
    eng.close()


def test_same_seed_same_bytes_and_batch_invariance(mini_ref, L):
    def run(splits, seed):
        eng, _, _ = pc.make_engine("guppy", mini_ref, fastq=True, seed=seed)
        out = []
        start = 0
        for n in splits:
            eng.simulate(L.NS_KIND_ALIGNED, start, n)
            b = eng.fetch()
            out += [(b.read_seq(i), b.read_qual(i).tobytes()) for i in range(n)]
            start += n
        eng.close()
        return out
    a = run([600], 42)
    assert a == run([600], 42)
    assert a == run([100, 37, 463], 42)            # read i depends on (seed, i) only
    assert a != run([600], 43)


def test_zero_reads_and_state_errors(mini_ref, L):
    from nanosim_b200.engine import Engine, NanoSimError
    eng = Engine(0, 1)
    with pytest.raises(NanoSimError):
        eng.simulate(L.NS_KIND_ALIGNED, 0, 10)         # nothing configured yet
    eng.close()
    eng, _, _ = pc.make_engine("guppy", mini_ref, fastq=False, seed=1)
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, 0)
    assert info.n_reads == 0 and info.total_bases == 0
    with pytest.raises(NanoSimError):
        eng.configure(min_len=100, max_len=50)
    with pytest.raises(NanoSimError):
        eng.configure(perfect=True, chimeric=True)
    eng.close()


def test_min_max_length_window(mini_ref, L):
    eng, _, _ = pc.make_engine("guppy", mini_ref, fastq=False, seed=9, min_len=2000, max_len=6000)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 3000)
    b = eng.fetch()
    assert b.reads["seq_len"].min() >= 2000 and b.reads["seq_len"].max() <= 6000
    assert b.reads["attempts"].max() > 0              # the rejection loop (simulator.py:1367) actually ran
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 500)
    bu = eng.fetch()
    assert bu.reads["seq_len"].min() >= 2000 and bu.reads["seq_len"].max() <= 6000
    eng.close()


def test_device_op_stats_equal_host_stats(ecoli, L):
    eng, _, _ = pc.make_engine("guppy", ecoli, fastq=False, seed=2)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 3000)
    b = eng.fetch(want_ops=True)
    host = pc.batch_stats(b, ecoli, False)
    dev = eng.op_stats()
    assert dev["events"] == host["events"] and dev["event_bases"] == host["event_bases"]
    assert dev["ref_bases"] == host["ref_bases"]
    for k in ("mis", "ins", "del"):
        assert np.array_equal(dev["ev_len"][k], host["ev_len"][k])
    assert np.array_equal(dev["match_run"], host["match_run"]) and np.array_equal(dev["first_match"], host["first_match"])
    merged = pc.merge_op_stats(rs.empty(), dev, aligned_comp=True)
    for k in ("events_per_read", "mis_sub", "ins_base", "base_comp_aligned"):
        assert host[k].sum() > 0 and np.array_equal(merged[k], host[k]), k
    eng.close()


@pytest.mark.parametrize("model,chim", [("guppy", False), ("dorado", True)])
def test_statistics_vs_oracle_small(model, chim, mini_ref, L, tmp_path):
    """Oracle = pure-Python restatement, a few hundred reads (seconds); device = 30k reads.  Loose tolerances sized
    to the oracle's sampling noise."""
    import nanosim_oracle as no
    eng, cm, t = pc.make_engine(model, mini_ref, fastq=True, chimeric=chim, seed=17)
    s_dev = rs.empty()
    eng.simulate(L.NS_KIND_ALIGNED, 0, 30000)
    pc.batch_stats(eng.fetch(want_ops=True), mini_ref, True, s_dev)
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 3000)
    pc.batch_stats(eng.fetch(), mini_ref, True, s_dev)
    eng.close()
    recs = no.read_fasta(os.path.join(GOLDEN, "mini_ref.fa"))
    s_or = pc.oracle_stats(cm, recs, 500 if model == "guppy" else 250, 150, True, chimeric=chim, tmpdir=str(tmp_path))
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.04 if model == "guppy" else 0.08, p_min=1e-5, label=model)
    for k in ("qual_middle", "qual_ht", "qual_unaligned"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        if p < 1e-5:
            fails.append("%s %s chi2 %.1f dof %d p %.3g" % (model, k, st, dof, p))
    fr_dev = s_dev["strand_R_aligned"] / s_dev["n_aligned"]
    assert abs(fr_dev - (1 - t.strandness)) < 0.02
    assert not fails, "\n".join(fails)


def _device_run_stats(eng, ref, L, n_aligned, n_unaligned, batch, fastq):
    s = rs.empty()
    for start in range(0, n_aligned, batch):
        n = min(batch, n_aligned - start)
        eng.simulate(L.NS_KIND_ALIGNED, start, n)
        b = eng.fetch(want_ops=False)
        pc.meta_stats(b, s)
        pc.merge_op_stats(s, eng.op_stats(), aligned_comp=True)
    for start in range(0, n_unaligned, batch):
        n = min(batch, n_unaligned - start)
        eng.simulate(L.NS_KIND_UNALIGNED, start, n)
        pc.meta_stats(eng.fetch(want_ops=False), s)
    return s


def test_vs_unmodified_reference_1M_reads(ecoli, L):
    """BASELINE config-1 reference/model at 1M reads, against histograms of the unmodified reference
    (tests/golden/ref_stats_guppy_fasta.json).  north_star: per-base edit-type counts within +-0.1 %."""
    path = os.path.join(GOLDEN, "ref_stats_guppy_fasta.json")
    gold, meta = pc.golden(path)
    n_al, n_un = int(gold["n_aligned"]), int(gold["n_unaligned"])
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=False, seed=2024)
    s = _device_run_stats(eng, ecoli, L, n_al, n_un, 125000, False)
    eng.close()
    rd, rg = pc.rates(s), pc.rates(gold)
    print("per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    # the reference's own chunk-to-chunk noise bounds what +-0.1 % can mean
    # north_star: identical read-length and per-read error-count histograms, per-base edit-type counts within +-0.1 %
    fails = pc.compare_stats(s, gold, rate_tol=1e-3, p_min=1e-6, label="1M",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match",
                                   "events_per_read"])
    # which base a mismatch / an insertion produces (simulator.py:1968-1973, 1989-1991) and the reads' composition
    fails += pc.compare_base_choices(s, gold, 1e-6, label="1M")
    # unaligned lengths: the reference forks its unaligned workers WITHOUT reseeding numpy (simulator.py:1648-1660), so
    # with -t 8 all eight workers draw the same KDE lengths (8-fold duplicated sample).  They are compared against a
    # separate golden run made of independent -t 1 processes.
    g1, _ = pc.golden(os.path.join(GOLDEN, "ref_stats_guppy_fasta_t1.json"))
    assert s["len_unaligned"].sum() > 0 and g1["len_unaligned"].sum() > 0
    st, dof, p = pc.chi2_two_sample(s["len_unaligned"], g1["len_unaligned"])
    print("len_unaligned vs -t 1 golden: chi2 %.1f dof %d p %.3g" % (st, dof, p))
    if p < 1e-6:
        fails.append("1M histogram len_unaligned (vs -t 1 golden): chi2 %.1f dof %d p %.3g" % (st, dof, p))
    fr_d, fr_g = s["strand_R_unaligned"] / s["n_unaligned"], g1["strand_R_unaligned"] / g1["n_unaligned"]
    assert abs(fr_d - fr_g) < 0.02
    mean_dev, mean_ref = s["aligned_bases"] / s["n_aligned"], gold["aligned_bases"] / gold["n_aligned"]
    assert abs(mean_dev / mean_ref - 1) < 5e-3, (mean_dev, mean_ref)
    assert abs(s["strand_R_aligned"] / s["n_aligned"] - gold["strand_R_aligned"] / gold["n_aligned"]) < 3e-3
    assert not fails, "\n".join(fails)


def _run_with_quals(eng, ref, L, n_al, n_un, batch):
    s = rs.empty()
    for start in range(0, n_al, batch):
        n = min(batch, n_al - start)
        eng.simulate(L.NS_KIND_ALIGNED, start, n)
        pc.batch_stats(eng.fetch(want_ops=False), ref, True, s)      # lengths, strands, quality histograms
        pc.merge_op_stats(s, eng.op_stats())                           # event histograms on the device
    for start in range(0, n_un, batch):
        n = min(batch, n_un - start)
        eng.simulate(L.NS_KIND_UNALIGNED, start, n)
        pc.batch_stats(eng.fetch(), ref, True, s)
    return s


def test_vs_unmodified_reference_dorado_fastq_chimeric(ecoli, L):
    """100k reads of `simulator.py genome --fastq --chimeric` with the dorado kit-v14 model (unmodified reference) vs
    the device: chimeric fraction, segments per read, per-base rates, length/event/quality histograms."""
    path = os.path.join(GOLDEN, "ref_stats_dorado_fastq_chimeric.json")
    gold, _ = pc.golden(path)
    eng, cm, t = pc.make_engine("dorado", ecoli, fastq=True, chimeric=True, seed=77)
    s = _run_with_quals(eng, ecoli, L, int(gold["n_aligned"]), int(gold["n_unaligned"]), 25000)
    eng.close()
    rd, rg = pc.rates(s), pc.rates(gold)
    print("dorado per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    fails = pc.compare_stats(s, gold, rate_tol=2.5e-3, p_min=1e-6, label="dorado",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    for k in ("qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s[k], gold[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-6:
            fails.append("dorado %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    fc_d, fc_g = s["n_chimeric"] / s["n_aligned"], gold["n_chimeric"] / gold["n_aligned"]
    assert abs(fc_d - fc_g) < 4 * np.sqrt(fc_g / gold["n_aligned"]) + 1e-4, (fc_d, fc_g)
    assert abs(s["n_segments"] / s["n_aligned"] - gold["n_segments"] / gold["n_aligned"]) < 3e-3
    assert abs(s["aligned_bases"] / s["n_aligned"] / (gold["aligned_bases"] / gold["n_aligned"]) - 1) < 1.5e-2
    assert not fails, "\n".join(fails)


def test_qualities_vs_unmodified_reference_guppyq(ecoli, L):
    """50k FASTQ reads of the unmodified reference with the config-2 model (guppy + dorado quality table): quality
    histograms of aligned middles (match/mis/ins mixture), head/tail regions and unaligned reads."""
    path = os.path.join(GOLDEN, "ref_stats_guppyq_fastq.json")
    gold, _ = pc.golden(path)
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=True, seed=78)
    s = _run_with_quals(eng, ecoli, L, int(gold["n_aligned"]), int(gold["n_unaligned"]), 25000)
    eng.close()
    fails = pc.compare_stats(s, gold, rate_tol=3e-3, p_min=1e-6, label="guppyq",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    # unaligned qualities: with -t 8 the reference's unaligned workers share one numpy stream (simulator.py:1648-1660),
    # i.e. identical quality draws in all eight workers; they are compared with independent -t 1 processes instead.
    g1, _ = pc.golden(os.path.join(GOLDEN, "ref_stats_guppyq_fastq_t1.json"))
    for k, g in (("qual_middle", gold), ("qual_ht", gold), ("qual_unaligned", g1)):
        assert s[k].sum() > 0 and g[k].sum() > 0, k
        st, dof, p = pc.chi2_two_sample(s[k], g[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-6:
            fails.append("guppyq %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    assert not fails, "\n".join(fails)


def _hp_reference(n_chrom=3, size=40000, seed=11):
    """ACGT-only reference rich in homopolymer runs (4..14) so that the -hp/-k paths are exercised on every read."""
    from nanosim_b200.reference_fasta import PackedReference
    rng = np.random.default_rng(seed)
    recs = []
    for c in range(n_chrom):
        s = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size)].copy()
        for _ in range(size // 60):
            p = int(rng.integers(0, size - 20))
            s[p:p + int(rng.integers(4, 15))] = b"ACGT"[int(rng.integers(0, 4))]
        recs.append(("hp%d" % c, s))
    return PackedReference.from_records(recs), [(n, a.tobytes().decode()) for n, a in recs]


def _in_hp_mask(seg, k):
    change = np.flatnonzero(seg[1:] != seg[:-1])
    bounds = np.concatenate([[0], change + 1, [len(seg)]])
    runs = np.diff(bounds)
    return np.repeat(runs >= k, runs)


def test_homopolymer_scripts_bit_exact_and_filter_invariant(L):
    """-hp -k 6: (1) the rewritten scripts (COPY / reference skips / literals) reproduce the device's bases exactly;
    (2) no surviving error event touches a homopolymer run of the unmutated segment (simulator.py:1929-1947)."""
    ref, _ = _hp_reference()
    eng, cm, t = pc.make_engine("dorado", ref, fastq=True, chimeric=True, kmer_bias=6, seed=13)
    info = eng.simulate(L.NS_KIND_ALIGNED, 0, 1200)
    b = eng.fetch(want_ops=True)
    assert pc.check_edit_scripts(b, ref, True) > 0
    assert ((b.ops[:0] >> 28) == 5).sum() == 0
    ref_off = ref.offsets.astype(np.int64)
    n_events = n_lit = 0
    for pcs in b.pieces[b.pieces["kind"] == L.NS_PIECE_SEGMENT]:
        assert int(pcs["ev_off"]) != int(pcs["op_off"])
        seg = ref.bases[int(ref_off[pcs["chrom"]]) + int(pcs["pos"]): int(ref_off[pcs["chrom"]]) + int(pcs["pos"]) + int(pcs["ref_len"])]
        mask = _in_hp_mask(seg, 6)
        ty, ln, out_adv, ref_adv, out_start, ref_start = pc._piece_layout(b, pcs, events=True)
        for j in np.nonzero((ty >= 1) & (ty <= 3))[0]:
            lo = int(ref_start[j]) - (1 if ty[j] == 2 else 0)
            hi = int(ref_start[j]) + int(ln[j]) - 1
            assert not mask[max(lo, 0):min(hi, len(mask) - 1) + 1].any(), "event inside a homopolymer survived"
            n_events += 1
        o = b.ops[int(pcs["op_off"]): int(pcs["op_off"]) + int(pcs["n_ops"])]
        n_lit += int(((o >> 28) == 5).sum())
    assert n_events > 1000 and n_lit > 1000
    eng.close()


def test_homopolymer_statistics_vs_oracle(L, tmp_path):
    """mutate_homo + the error filter against the pure-Python oracle on a homopolymer-rich reference."""
    ref, recs = _hp_reference(size=60000)
    eng, cm, t = pc.make_engine("dorado", ref, fastq=True, kmer_bias=6, seed=19)
    s_dev = rs.empty()
    eng.simulate(L.NS_KIND_ALIGNED, 0, 20000)
    pc.batch_stats(eng.fetch(want_ops=True), ref, True, s_dev)
    eng.close()
    s_or = pc.oracle_stats(cm, recs, 220, 0, True, tmpdir=str(tmp_path), kmer_bias=6)
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.08, p_min=1e-5, label="hp",
                             keys=["len_aligned", "len_middle_ref", "match_run", "first_match"])
    for k in ("hp_runs", "qual_middle"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-5:
            fails.append("hp %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    # net length change of the pass: mean read length relative to the aligned region, device vs oracle
    rd = (s_dev["aligned_bases"] - s_dev["head_bases"] - s_dev["tail_bases"]) / s_dev["ref_bases"]
    ro = (s_or["aligned_bases"] - s_or["head_bases"] - s_or["tail_bases"]) / s_or["ref_bases"]
    print("middle bases per reference base: device %.5f oracle %.5f" % (rd, ro))
    assert abs(rd / ro - 1) < 3e-3, (rd, ro)
    assert not fails, "\n".join(fails)


def test_homopolymer_vs_unmodified_reference(ecoli, L):
    """50k reads of `simulator.py genome --fastq --chimeric -hp -k 6` (dorado model, unmodified reference)."""
    path = os.path.join(GOLDEN, "ref_stats_dorado_fastq_hp6_chimeric.json")
    gold, _ = pc.golden(path)
    assert "hp_runs" in gold, "golden file predates the homopolymer histogram: regenerate it"
    eng, cm, t = pc.make_engine("dorado", ecoli, fastq=True, chimeric=True, kmer_bias=6, seed=79)
    s = _run_with_quals(eng, ecoli, L, int(gold["n_aligned"]), int(gold["n_unaligned"]), 25000)
    eng.close()
    rd, rg = pc.rates(s), pc.rates(gold)
    print("hp per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    fails = pc.compare_stats(s, gold, rate_tol=4e-3, p_min=1e-6, label="hp6",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    for k in ("hp_runs", "qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s[k], gold[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-6:
            fails.append("hp6 %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    md = (s["aligned_bases"] - s["head_bases"] - s["tail_bases"]) / s["ref_bases"]
    mg = (gold["aligned_bases"] - gold["head_bases"] - gold["tail_bases"]) / gold["ref_bases"]
    print("middle bases per reference base: device %.6f reference %.6f" % (md, mg))
    assert abs(md / mg - 1) < 1e-3
    assert not fails, "\n".join(fails)


@pytest.fixture(scope="module")
def meta_ref():
    from conftest import meta_fixture
    from nanosim_b200.reference_fasta import MetaReference, read_abundance
    meta_fixture()                                   # writes genome_list_local.tsv with this checkout's paths
    meta = os.path.join(GOLDEN, "meta")
    ref = MetaReference.from_genome_list(os.path.join(meta, "genome_list_local.tsv"), os.path.join(meta, "dna_type.tsv"))
    numbers, samples = read_abundance(os.path.join(meta, "abundance.tsv"), ref.species)
    return ref, numbers, samples


def _species_base_fractions(b, ref, L):
    seg = b.pieces[b.pieces["kind"] == L.NS_PIECE_SEGMENT]
    sp = ref.chrom_species[seg["chrom"]]
    tot = np.bincount(sp, weights=seg["ref_len"].astype(np.float64), minlength=len(ref.species))
    return tot / tot.sum()


def test_metagenome_scripts_strand_and_quota(meta_ref, L):
    """Metagenome mode on four species (linear + circular chromosomes): bit-exact scripts, one strand per batch
    (simulator.py:860), per-chromosome circular wrap, species base composition follows the abundance quotas (:772-775)."""
    ref, numbers, samples = meta_ref
    eng, cm, t = pc.make_meta_engine(ref, samples[0], fastq=True, chimeric=True, seed=23)
    fr_all = np.zeros(len(ref.species))
    strands = set()
    for k in range(3):
        eng.simulate(L.NS_KIND_ALIGNED, k * 4000, 4000)
        b = eng.fetch(want_ops=True)
        assert pc.check_edit_scripts(b, ref, True, max_reads=1500) > 0
        assert len(set(b.reads["reversed"].tolist())) == 1          # is_reversed is drawn once per batch
        strands.add(int(b.reads["reversed"][0]))
        fr_all += _species_base_fractions(b, ref, L)
        seg = b.pieces[b.pieces["kind"] == L.NS_PIECE_SEGMENT]
        lin = ref.chrom_circular[seg["chrom"]] == 0
        assert ((seg["pos"].astype(np.int64) + seg["ref_len"])[lin] <= ref.lengths[seg["chrom"]][lin]).all()
    want = np.asarray(samples[0]) / np.sum(samples[0])
    print("species base fractions", fr_all / 3, "abundance", want)
    assert np.abs(fr_all / 3 - want).max() < 0.01
    assert (b.reads["n_pieces"] > 1).any()
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 6000)
    bu = eng.fetch()
    cnt = np.bincount(ref.chrom_species[bu.pieces["chrom"]], minlength=len(ref.species)) / len(bu.pieces)
    print("unaligned species fractions", cnt)          # uniform species choice (:1705-1706), then rejection by length
    assert cnt.min() > 0.1
    eng.close()


def test_metagenome_statistics_vs_oracle(meta_ref, L, tmp_path):
    """simulation_aligned_metagenome of the pinned oracle (a few hundred reads) vs the device."""
    import nanosim_oracle as no
    from conftest import meta_fixture, oracle_model
    ref, numbers, samples = meta_ref
    eng, cm, t = pc.make_meta_engine(ref, samples[0], fastq=True, chimeric=True, seed=29)
    s_dev = rs.empty()
    fr = np.zeros(len(ref.species))
    for k in range(4):
        eng.simulate(L.NS_KIND_ALIGNED, k * 5000, 5000)
        b = eng.fetch(want_ops=True)
        pc.batch_stats(b, ref, True, s_dev)
        fr += _species_base_fractions(b, ref, L) / 4
    eng.close()
    oref, onum, omulti = meta_fixture()
    m = oracle_model(cm, tmp_path, fastq=True, chimeric=True, mode="metagenome")
    abun = omulti["sample0"]
    infl = {sp: no.inflate_abun(abun, sp, m.abun_inflation) for sp in abun}
    import random
    random.seed(77)
    np.random.seed(77)
    sink = no.ReadSink()
    no.simulation_aligned_metagenome(oref, m, sink, abun, infl, 50, max(oref.max_chrom.values()), None, True, 450, False, True)
    prefix = os.path.join(str(tmp_path), "ometa")
    with open(prefix + "_aligned_reads.fastq", "w") as f:
        f.write(no.format_records(sink.records, True))
    with open(prefix + "_aligned_error_profile", "w") as f:
        f.write("Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n")
        f.writelines(r + "\n" for r in sink.error_rows)
    s_or = rs.stats_from_prefix(prefix, True)
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.05, p_min=1e-5, label="meta",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    for k in ("qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-5:
            fails.append("meta %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    fc_d, fc_o = s_dev["n_chimeric"] / s_dev["n_aligned"], s_or["n_chimeric"] / s_or["n_aligned"]
    assert abs(fc_d - fc_o) < 0.035, (fc_d, fc_o)
    # species composition of the oracle run from its read names ({species}-{chrom}_{pos};...)
    tot = {sp: 0 for sp in abun}
    for name, seq, q in sink.records:
        parts = name.rsplit("_", 4)
        lens = [int(x) for x in parts[3].split(";")]
        locs = [c for c in parts[0].split("_aligned_")[0].split(";") if not c.startswith("gap_")]
        for loc, n in zip(locs, lens):
            tot[[sp for sp in abun if loc.startswith(sp + "-")][0]] += n
    fo = np.asarray([tot[sp] for sp in ref.species], dtype=np.float64)
    fo /= fo.sum()
    print("species base fractions device", fr, "oracle", fo)
    assert np.abs(fr - fo).max() < 0.03
    assert not fails, "\n".join(fails)


def test_cli_metagenome_end_to_end(meta_ref, tmp_path, L):
    from nanosim_b200 import simulator
    meta = os.path.join(GOLDEN, "meta")
    out = os.path.join(str(tmp_path), "mg")
    simulator.main(["metagenome", "-gl", os.path.join(meta, "genome_list_local.tsv"), "-a", os.path.join(meta, "abundance.tsv"),
                    "-dl", os.path.join(meta, "dna_type.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["even"]), "-o", out,
                    "--fastq", "--chimeric", "--seed", "3"])
    for i, n in enumerate((300, 200)):
        s = rs.stats_from_prefix(out + "_sample%d" % i, True)
        assert s["n_aligned"] + s["n_unaligned"] == n
        first = open(out + "_sample%d_aligned_reads.fastq" % i).readline()
        assert first.startswith("@") and "-" in first and "_aligned_" in first
    chim = [l for l in open(out + "_sample0_aligned_reads.fastq") if l.startswith("@") and "_chimeric_" in l]
    assert all(";gap_" in l for l in chim)


@pytest.fixture(scope="module")
def trx_ref():
    from nanosim_b200.reference_fasta import PackedReference, read_expression, read_polya_list
    T = os.path.join(GOLDEN, "trx")
    ref = PackedReference.from_fasta(os.path.join(T, "transcripts.fa"))
    chrom, w = read_expression(os.path.join(T, "expression.tsv"), ref)
    return ref, chrom, w, read_polya_list(os.path.join(T, "polya.txt"), ref)


def test_transcriptome_scripts_polya_uracil(trx_ref, L):
    """Transcriptome mode (--no_model_ir): bit-exact scripts, reads inside their transcript, polyA rule
    (simulator.py:1689), T->U, expressed transcripts only."""
    from nanosim_b200.reference_fasta import POLYA_SCALE
    ref, chrom, w, polya = trx_ref
    eng, cm, t = pc.make_trx_engine(ref, chrom, w, polya, fastq=True, seed=41, polya_scale=POLYA_SCALE["guppy"])
    eng.simulate(L.NS_KIND_ALIGNED, 0, 6000)
    b = eng.fetch(want_ops=True)
    assert pc.check_edit_scripts(b, ref, True) > 0
    pcs = b.pieces
    tlen = ref.lengths[pcs["chrom"]]
    assert set(np.unique(pcs["chrom"]).tolist()) <= set(chrom.tolist())
    assert (pcs["pos"].astype(np.int64) + pcs["ref_len"] <= tlen).all()
    near_end = pcs["pos"].astype(np.int64) + pcs["ref_len"] + 10 >= tlen
    flagged = polya[pcs["chrom"]] == 1
    assert ((pcs["polya_len"] > 0) <= (near_end & flagged)).all()          # a tail only where the rule allows one
    assert (pcs["polya_len"][near_end & flagged] >= 2).all()               # int(expon(loc=2)) >= 2
    mean_tail = pcs["polya_len"][near_end & flagged].mean()
    assert abs(mean_tail - (2 + POLYA_SCALE["guppy"] - 0.5)) < 0.4, mean_tail
    fr = b.reads["reversed"].mean()
    assert fr < 0.03                                                        # dRNA strandness 0.994
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 1500)
    bu = eng.fetch()
    assert (bu.pieces["pos"].astype(np.int64) + bu.pieces["ref_len"] <= ref.lengths[bu.pieces["chrom"]]).all()
    assert (bu.pieces["ref_len"] < ref.lengths[bu.pieces["chrom"]]).all()  # `if length < seq_len[key]` (:1698)
    eng.close()
    eng, _, _ = pc.make_trx_engine(ref, chrom, w, None, fastq=False, seed=41, uracil=True)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 500)
    bq = eng.fetch()
    used = np.concatenate([bq.seq[int(r["seq_off"]):int(r["seq_off"]) + int(r["seq_len"])] for r in bq.reads])
    assert (used != ord("T")).all() and (used == ord("U")).any()
    assert (bq.pieces["polya_len"] == 0).all()
    eng.close()


def test_transcriptome_statistics_vs_oracle(trx_ref, L, tmp_path):
    """simulation_aligned_transcriptome of the pinned oracle (600 reads, 2-D KDE sample of 600 rows) vs the device with the
    same sample size: the aligned-length-given-transcript law (select_nearest_kde2d), transcript usage, error rates."""
    import random
    import nanosim_oracle as no
    from conftest import oracle_model
    from nanosim_b200.reference_fasta import POLYA_SCALE
    ref, chrom, w, polya = trx_ref
    N = 600
    eng, cm, t = pc.make_trx_engine(ref, chrom, w, polya, fastq=True, seed=43, polya_scale=POLYA_SCALE["guppy"], kde2d_sample=N)
    s_dev = rs.empty()
    eng.simulate(L.NS_KIND_ALIGNED, 0, 40000)
    b = eng.fetch(want_ops=True)
    pc.batch_stats(b, ref, True, s_dev)
    use_dev = np.bincount(b.pieces["chrom"], minlength=len(ref.names)).astype(np.float64)
    frac_dev = (b.pieces["ref_len"] / ref.lengths[b.pieces["chrom"]])
    eng.close()
    T = os.path.join(GOLDEN, "trx")
    oref = no.OracleTrxReference.from_files(os.path.join(T, "transcripts.fa"), os.path.join(T, "expression.tsv"),
                                            os.path.join(T, "polya.txt"))
    m = oracle_model(cm, tmp_path, fastq=True)
    s_or = rs.empty()
    use_or = np.zeros(len(ref.names))
    frac_or = []
    for rep in range(3):                                    # three independent workers of N reads each
        random.seed(500 + rep)
        np.random.seed(500 + rep)
        sink = no.ReadSink()
        no.simulation_aligned_transcriptome(oref, m, sink, None, "guppy", N, True, True, False, False)
        prefix = os.path.join(str(tmp_path), "otrx%d" % rep)
        with open(prefix + "_aligned_reads.fastq", "w") as f:
            f.write(no.format_records(sink.records, True))
        with open(prefix + "_aligned_error_profile", "w") as f:
            f.write("Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n")
            f.writelines(r + "\n" for r in sink.error_rows)
        rs.merge(s_or, rs.stats_from_prefix(prefix, True))
        for name, seq, q in sink.records:
            trx = name.split("_")[0]
            i = ref.names.index(trx)
            use_or[i] += 1
            frac_or.append(int(name.rsplit("_", 4)[3]) / ref.lengths[i])
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.06, p_min=1e-5, label="trx",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    st, dof, p = pc.chi2_two_sample(use_dev, use_or)
    print("transcript usage chi2 %.1f dof %d p %.3g" % (st, dof, p))
    if p < 1e-5:
        fails.append("transcript usage chi2 %.1f dof %d p %.3g" % (st, dof, p))
    edges = np.linspace(0, 1.0001, 21)
    st, dof, p = pc.chi2_two_sample(np.histogram(frac_dev, edges)[0], np.histogram(frac_or, edges)[0])
    print("aligned fraction of transcript chi2 %.1f dof %d p %.3g" % (st, dof, p))
    if p < 1e-5:
        fails.append("aligned/transcript length ratio chi2 %.1f dof %d p %.3g" % (st, dof, p))
    assert not fails, "\n".join(fails)


def test_cli_transcriptome_end_to_end(trx_ref, tmp_path, L):
    from nanosim_b200 import simulator
    T = os.path.join(GOLDEN, "trx")
    out = os.path.join(str(tmp_path), "tx")
    simulator.main(["transcriptome", "-rt", os.path.join(T, "transcripts.fa"), "-e", os.path.join(T, "expression.tsv"),
                    "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", "800", "-o", out, "--no_model_ir", "--fastq",
                    "--polya", os.path.join(T, "polya.txt"), "-b", "guppy", "--seed", "5"])
    s = rs.stats_from_prefix(out, True)
    assert s["n_aligned"] + s["n_unaligned"] == 800 and s["n_aligned"] == int(round(800 * 1.6565173181434516 / 2.6565173181434516))
    first = open(out + "_aligned_reads.fastq").readline()
    assert first.startswith("@ENST") and "_aligned_0_" in first
    with pytest.raises(SystemExit):
        simulator.main(["transcriptome", "-rt", os.path.join(T, "transcripts.fa"), "-e", os.path.join(T, "expression.tsv"),
                        "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", "10", "-o", out, "--polya", os.path.join(T, "polya.txt")])


def _by_chrom(path, fastq):
    sys.path.insert(0, GOLDEN)
    from make_golden_runs_modes import by_chrom
    return by_chrom(path, fastq)


def _share_diff(a, b):
    keys = sorted(set(a) | set(b))
    va = np.array([a.get(k, 0) for k in keys], dtype=np.float64)
    vb = np.array([b.get(k, 0) for k in keys], dtype=np.float64)
    return keys, va, vb, np.abs(va / va.sum() - vb / vb.sum()).max()


def test_transcriptome_vs_unmodified_reference(trx_ref, tmp_path, L):
    """400k reads of the unmodified `simulator.py transcriptome --no_model_ir -b guppy --polya ... -n 8000 -t 8` (50 runs,
    tests/golden/make_golden_runs_modes.py) against this CLI: same files, same parser.  -t is chosen so that the 2-D
    length-KDE sample has the reference's 623 rows per worker."""
    from nanosim_b200 import simulator
    path = os.path.join(GOLDEN, "ref_stats_trx_drna_fasta.json")
    gold, _ = pc.golden(path)
    T = os.path.join(GOLDEN, "trx")
    out = os.path.join(str(tmp_path), "tx")
    n = 200000
    simulator.main(["transcriptome", "-rt", os.path.join(T, "transcripts.fa"), "-e", os.path.join(T, "expression.tsv"),
                    "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", str(n), "-o", out, "--no_model_ir",
                    "--polya", os.path.join(T, "polya.txt"), "-b", "guppy", "--seed", "17", "-t", str(n // 8000 * 8)])
    s = rs.stats_from_prefix(out, False)
    rd, rg = pc.rates(s), pc.rates(gold)
    print("trx per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    fails = pc.compare_stats(s, gold, rate_tol=3e-3, p_min=1e-6, label="trx",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match",
                                   "len_unaligned", "events_per_read"])
    reads, bases = _by_chrom(out + "_aligned_reads.fasta", False)
    keys, va, vb, _ = _share_diff(reads, gold["by_chrom_reads"])
    st, dof, p = pc.chi2_two_sample(va, vb)
    print("reads per transcript: chi2 %.1f dof %d p %.3g" % (st, dof, p))
    if p < 1e-6:
        fails.append("trx reads per transcript chi2 %.1f dof %d p %.3g" % (st, dof, p))
    kb, ba, bb, d = _share_diff(bases, gold["by_chrom_bases"])
    print("max |share| difference of bases per transcript %.4g" % d)
    for j in np.argsort(-np.abs(ba / ba.sum() - bb / bb.sum()))[:6]:
        k = kb[j]
        print("  %s base share %.5f vs %.5f; reads %d vs %d; mean read %.1f vs %.1f" % (
            k, ba[j] / ba.sum(), bb[j] / bb.sum(), reads.get(k, 0), gold["by_chrom_reads"].get(k, 0),
            ba[j] / max(reads.get(k, 0), 1), bb[j] / max(gold["by_chrom_reads"].get(k, 0), 1)))
    # the reference reuses one 2-D KDE sample until a transcript repeats (simulator.py:1087-1090), which makes a transcript
    # whose nearest row is too long stay blocked for the life of that sample; the device draws the nearest row afresh
    # per attempt (DESIGN.md, deviations).  On this 71-transcript fixture the effect is at its largest.
    if d > 1e-2:
        fails.append("trx bases per transcript: share differs by %.4g" % d)
    fr = s["strand_R_aligned"] / s["n_aligned"], gold["strand_R_aligned"] / gold["n_aligned"]
    assert abs(fr[0] - fr[1]) < 2e-3, fr
    assert not fails, "\n".join(fails)


def test_metagenome_vs_unmodified_reference(meta_ref, tmp_path, L):
    """200k reads of the unmodified `simulator.py metagenome --fastq --chimeric` (Even model, 10 runs of 20000, -t 8)
    against this CLI on the same 4-species fixture: histograms, rates, qualities, species and chromosome shares."""
    from nanosim_b200 import simulator
    path = os.path.join(GOLDEN, "ref_stats_meta_even_fastq_chimeric.json")
    gold, _ = pc.golden(path)
    meta = os.path.join(GOLDEN, "meta")
    ab = os.path.join(str(tmp_path), "abun.tsv")
    with open(os.path.join(meta, "abundance.tsv")) as f, open(ab, "w") as o:
        f.readline()
        o.write("Size\t40000\n")
        for line in f:
            pp = line.rstrip("\n").split("\t")
            o.write("%s\t%s\n" % (pp[0], pp[1]))
    out = os.path.join(str(tmp_path), "mg")
    simulator.main(["metagenome", "-gl", os.path.join(meta, "genome_list_local.tsv"), "-a", ab, "-dl", os.path.join(meta, "dna_type.tsv"),
                    "-c", os.path.join(pc.DATA, pc.MODELS["even"]), "-o", out, "--fastq", "--chimeric", "--seed", "23",
                    "--batch_reads", "20000"])
    s = rs.stats_from_prefix(out + "_sample0", True)
    rd, rg = pc.rates(s), pc.rates(gold)
    print("meta per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    fails = pc.compare_stats(s, gold, rate_tol=3e-3, p_min=1e-6, label="meta",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match", "events_per_read"])
    for k in ("qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s[k], gold[k])
        print(k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-6:
            fails.append("meta %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    reads, bases = _by_chrom(out + "_sample0_aligned_reads.fastq", True)
    sp = lambda d: {k2: sum(v for k, v in d.items() if k.split("-")[0] == k2) for k2 in {k.split("-")[0] for k in d}}
    _, va, vb, d_sp = _share_diff(sp(bases), sp(gold["by_chrom_bases"]))
    _, _, _, d_ch = _share_diff(reads, gold["by_chrom_reads"])
    print("species base shares device", va / va.sum(), "reference", vb / vb.sum(), "max diff %.4g; chromosome read shares max diff %.4g" % (d_sp, d_ch))
    if d_sp > 0.01:
        fails.append("meta species base shares differ by %.4g" % d_sp)
    if d_ch > 0.01:
        fails.append("meta chromosome read shares differ by %.4g" % d_ch)
    fc = s["n_chimeric"] / s["n_aligned"], gold["n_chimeric"] / gold["n_aligned"]
    if abs(fc[0] / fc[1] - 1) > 0.06:
        fails.append("meta chimeric fraction %.4f vs %.4f" % fc)
    assert not fails, "\n".join(fails)


def test_host_formatters_match_python_on_device_batches(mini_ref, L):
    """ns_format_names / ns_format_error_profile (what the CLI writes) against the readable Python implementations on real
    batches: chimeric dorado reads with the homopolymer pass (event bases fixed by the device), guppy reads."""
    from nanosim_b200.records import error_profile_rows, format_error_profile, name_table, read_names
    for model, kw in (("dorado", {"chimeric": True, "kmer_bias": 6}), ("guppy", {})):
        eng, cm, t = pc.make_engine(model, mini_ref, fastq=True, seed=61, **kw)
        eng.simulate(L.NS_KIND_ALIGNED, 40, 400)
        b = eng.fetch(want_ops=True)
        eng.close()
        names = read_names(b, mini_ref.names, 40)
        tab = name_table(b, mini_ref.names, 40)
        assert tab.tolist() == names
        want = "".join(error_profile_rows(b, names, mini_ref, seed=61)).encode()
        assert format_error_profile(b, tab, mini_ref, seed=61, n_threads=4) == want and len(want) > 10000


def test_cli_output_is_independent_of_batching(ecoli, tmp_path, L):
    """Many small batches through the overlapped pipeline (contexts pull jobs as they free up, results are consumed in
    submission order) write byte-identical files to one big batch."""
    from nanosim_b200 import simulator
    ref = os.path.join(str(tmp_path), "ecoli5m.fa")
    synth.ecoli5m(ref)
    outs = []
    for tag, batch in (("a", "100000"), ("b", "173")):
        out = os.path.join(str(tmp_path), tag)
        simulator.main(["genome", "-rg", ref, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "3000", "-o", out, "--fastq",
                        "--seed", "12", "--batch_reads", batch, "-t", "3"])
        outs.append(out)
    for suffix in ("_aligned_reads.fastq", "_unaligned_reads.fastq", "_aligned_error_profile"):
        a, b = open(outs[0] + suffix, "rb").read(), open(outs[1] + suffix, "rb").read()
        assert a == b and len(a) > 1000, suffix


def test_perfect_reads_vs_unmodified_reference(ecoli, L):
    """100k reads of `simulator.py genome --perfect` (unmodified reference): length law (kde_aligned_reads within
    [min_l, max_l], :1285-1299), strand, no errors, no head/tail."""
    path = os.path.join(GOLDEN, "ref_stats_guppy_perfect.json")
    gold, _ = pc.golden(path)
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=False, perfect=True, seed=91)
    s = _device_run_stats(eng, ecoli, L, int(gold["n_aligned"]), 0, 50000, False)
    eng.close()
    assert s["head_bases"] == 0 and s["tail_bases"] == 0 and sum(s["events"].values()) == 0
    assert s["aligned_bases"] == s["ref_bases"]
    fails = []
    for k in ("len_aligned", "len_middle_ref"):
        st, dof, p = pc.chi2_two_sample(s[k], gold[k])
        print("perfect", k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-6:
            fails.append("perfect %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    assert abs(s["aligned_bases"] / s["n_aligned"] / (gold["aligned_bases"] / gold["n_aligned"]) - 1) < 1e-2
    assert abs(s["strand_R_aligned"] / s["n_aligned"] - gold["strand_R_aligned"] / gold["n_aligned"]) < 8e-3
    assert not fails, "\n".join(fails)


def test_med_sd_vs_unmodified_reference(ecoli, L):
    """100k reads of `simulator.py genome -med 5000 -sd 1.05` (unmodified reference).  The reference subtracts a head/tail
    remainder from a log-normal total and then filters the list, which breaks the pairing with the remainder a read
    later gets (:1285-1296); the device subtracts an independent remainder (DESIGN.md).  Read-level laws must agree."""
    path = os.path.join(GOLDEN, "ref_stats_guppy_medsd.json")
    gold, _ = pc.golden(path)
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=False, seed=93)
    eng.configure(fastq=False, min_len=50, max_len=ecoli.max_chrom, median_len=5000, sd_len=1.05)
    s = _device_run_stats(eng, ecoli, L, int(gold["n_aligned"]), int(gold["n_unaligned"]), 50000, False)
    eng.close()
    rd, rg = pc.rates(s), pc.rates(gold)
    print("med/sd per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    fails = pc.compare_stats(s, gold, rate_tol=4e-3, p_min=1e-6, label="medsd",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    st, dof, p = pc.chi2_two_sample(s["len_unaligned"], gold["len_unaligned"])
    print("med/sd len_unaligned chi2 %.1f dof %d p %.3g (the reference's -t 8 unaligned workers share one numpy stream)" % (st, dof, p))
    assert abs(s["aligned_bases"] / s["n_aligned"] / (gold["aligned_bases"] / gold["n_aligned"]) - 1) < 1.5e-2
    assert not fails, "\n".join(fails)


@pytest.fixture(scope="module")
def ir_fixture():
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.reference_fasta import PackedReference, read_expression, read_polya_list
    D = os.path.join(GOLDEN, "ir")
    trx = PackedReference.from_fasta(os.path.join(D, "transcripts.fa"))
    genome = PackedReference.from_fasta(os.path.join(D, "genome.fa"))
    ref = PackedReference.concat(trx, genome)
    chrom, w = read_expression(os.path.join(D, "expression.tsv"), trx)
    polya = np.concatenate([read_polya_list(os.path.join(D, "polya.txt"), trx), np.zeros(len(genome.names), dtype=np.uint8)])
    st = ir.TranscriptStructures.from_gff3(os.path.join(D, "annotation.gff3"), trx.names, genome.raw_names)
    irm = ir.IntronRetention(ir.read_ir_markov_model(os.path.join(D, "IR_markov_model")), st, trx.lengths, len(trx.names))
    return D, trx, genome, ref, chrom, w, polya, irm


def test_intron_retention_reemit(ir_fixture, L, monkeypatch):
    """Transcriptome reads that retain introns (simulator.py:1156-1183): the host half decides and lays them out on the genome,
    ns_reemit emits them again.  Untouched reads keep their bytes; patched reads keep length, qualities and every base
    that does not come from the reference; their scripts re-applied to the GENOME reproduce the bases bit-exactly (minus
    strand included); the intervals are the ones the pinned oracle extracts from the same uniforms."""
    import random
    import nanosim_oracle as no
    from nanosim_b200 import intron_retention as ir
    from nanosim_b200.records import error_profile_rows, format_error_profile, name_table, read_names
    from nanosim_b200.reference_fasta import POLYA_SCALE
    D, trx, genome, ref, chrom, w, polya, irm = ir_fixture
    seed = 71
    eng, cm, t = pc.make_trx_engine(ref, chrom, w, polya, fastq=True, seed=seed, polya_scale=POLYA_SCALE["guppy"],
                                    trx_records=len(trx.names), max_len=trx.max_chrom)
    eng.simulate(L.NS_KIND_ALIGNED, 500, 4000)
    b0 = eng.fetch(want_ops=True)
    assert (b0.pieces["chrom"] < len(trx.names)).all()
    patch = irm.plan_batch(b0.reads, b0.pieces, b0.ops, 500, seed, eng.info.n_pieces, eng.info.n_ops)
    assert patch is not None
    slots = patch[0]
    eng.reemit(*patch)
    b1 = eng.fetch(want_ops=True)
    assert 0.2 * 4000 < len(slots) < 0.95 * 4000                 # the fixture's IR model retains often
    assert pc.check_edit_scripts(b1, ref, True) > 0
    touched = np.zeros(4000, dtype=bool)
    touched[slots] = True
    oref = no.OracleTrxReference.from_files(os.path.join(D, "transcripts.fa"), os.path.join(D, "expression.tsv"), os.path.join(D, "polya.txt"))
    oref.load_ir(os.path.join(D, "genome.fa"), os.path.join(D, "annotation.gff3"), os.path.join(D, "IR_markov_model"))
    n_minus = n_named = 0
    for i in range(4000):
        a, n = int(b0.reads["seq_off"][i]), int(b0.reads["seq_len"][i])
        assert int(b1.reads["seq_len"][i]) == n and int(b1.reads["seq_off"][i]) == a
        assert np.array_equal(b0.qual[a:a + n], b1.qual[a:a + n])
        if not touched[i]:
            assert np.array_equal(b0.seq[a:a + n], b1.seq[a:a + n])
            continue
        p1 = b1.pieces[int(b1.reads["piece_first"][i]):int(b1.reads["piece_first"][i]) + int(b1.reads["n_pieces"][i])][::2]
        assert (p1["chrom"] >= len(trx.names)).all() and (p1["kind"] & L.NS_PIECE_GENOME).all()
        t0 = int(b0.pieces["chrom"][int(b0.reads["piece_first"][i])])
        key, n_int = trx.names[t0], int(irm.st.n_introns[t0])
        u = ir.ir_uniforms(seed, [500 + i], n_int + 1)[0]
        feed = iter(u[:n_int].tolist())
        monkeypatch.setattr(random, "random", lambda: next(feed))
        monkeypatch.setattr(random, "randint", lambda lo, hi: min(int(u[n_int] * (hi + 1)), hi) if hi > 0 else 0)
        flag, st_new = no.update_structure(oref.structure[key], oref.ir_model)
        assert flag
        ivs, _, ir_list = no.extract_read_pos(int(p1["ref_len"].sum()), oref.seq_len[key], st_new, False)
        got = sorted((int(x["pos"]), int(x["pos"]) + int(x["ref_len"])) for x in p1)
        assert got == [(s, e) for _, s, e, _ in ivs]
        assert sorted((int(x["pos"]), int(x["pos"]) + int(x["ref_len"])) for x in p1 if int(x["kind"]) & L.NS_PIECE_RETAINED) == [tuple(x) for x in ir_list]
        n_minus += bool(int(p1["kind"][0]) & L.NS_PIECE_REF_REV)
    names = read_names(b1, ref.names, 500, transcriptome=True)
    tab = name_table(b1, ref.names, 500, transcriptome=True)
    assert tab.tolist() == names
    n_named = sum("_RetainedIntron_" in x for x in names)
    assert n_minus > 50 and n_named > 100
    want = "".join(error_profile_rows(b1, names, ref, seed=seed)).encode()
    assert format_error_profile(b1, tab, ref, seed=seed, n_threads=4) == want
    eng.close()


def test_cli_transcriptome_with_intron_retention(ir_fixture, tmp_path, L):
    """The CLI with IR on (the reference's default): -rg genome, IR model and GFF3; output independent of the batch split."""
    from nanosim_b200 import simulator
    D = ir_fixture[0]
    outs = []
    for tag, batch in (("a", "100000"), ("b", "211")):
        out = os.path.join(str(tmp_path), tag)
        simulator.main(["transcriptome", "-rt", os.path.join(D, "transcripts.fa"), "-rg", os.path.join(D, "genome.fa"),
                        "-e", os.path.join(D, "expression.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", "1500", "-o", out,
                        "--fastq", "--polya", os.path.join(D, "polya.txt"), "-b", "guppy", "--seed", "9", "--batch_reads", batch,
                        "--ir_markov_model", os.path.join(D, "IR_markov_model"), "--ir_gff3", os.path.join(D, "annotation.gff3")])
        outs.append(out)
    for suffix in ("_aligned_reads.fastq", "_unaligned_reads.fastq", "_aligned_error_profile"):
        a, b = open(outs[0] + suffix, "rb").read(), open(outs[1] + suffix, "rb").read()
        assert a == b and len(a) > 1000, suffix
    heads = [l for l in open(outs[0] + "_aligned_reads.fastq") if l.startswith("@ENST")]
    assert sum("_RetainedIntron_" in h for h in heads) > 50
    s = rs.stats_from_prefix(outs[0], True)
    assert s["n_aligned"] + s["n_unaligned"] == 1500


def test_intron_retention_vs_unmodified_reference(ir_fixture, tmp_path, L):
    """96k reads of the unmodified `simulator.py transcriptome` with intron retention ON (its HTSeq / pysam calls served by the
    stand-ins of oracle/ref_shim.py) on the IR fixture, against this CLI: read-level histograms, error rates, the share
    of reads that retain an intron and how many retained intervals they cover."""
    from nanosim_b200 import simulator
    path = os.path.join(GOLDEN, "ref_stats_trx_ir_drna_fasta.json")
    gold, _ = pc.golden(path)
    D = ir_fixture[0]
    out = os.path.join(str(tmp_path), "ir")
    n = 96000
    simulator.main(["transcriptome", "-rt", os.path.join(D, "transcripts.fa"), "-rg", os.path.join(D, "genome.fa"),
                    "-e", os.path.join(D, "expression.tsv"), "-c", os.path.join(pc.DATA, pc.MODELS["drna"]), "-n", str(n), "-o", out,
                    "--polya", os.path.join(D, "polya.txt"), "-b", "guppy", "--seed", "29", "-t", str(n // 8000 * 8),
                    "--ir_markov_model", os.path.join(D, "IR_markov_model"), "--ir_gff3", os.path.join(D, "annotation.gff3")])
    s = rs.stats_from_prefix(out, False)
    rd, rg = pc.rates(s), pc.rates(gold)
    print("IR per-base rates device", rd, "reference", rg, "rel", {k: rd[k] / rg[k] - 1 for k in rd})
    # Two documented deviations show on this 16-transcript fixture where half of the reads retain an intron: (1) len_tail is
    # left out -- the name's last field is tail + polyA, and a retained-intron read keeps the polyA decision of its first
    # pass while the reference re-decides it from the genomic end of the last feature (simulator.py:186-189); (2) transcript
    # usage differs slightly (shared 2-D KDE sample, see test_transcriptome_vs_unmodified_reference), which moves the read
    # length mix and with it the per-base rates by a few 1e-3.
    fails = pc.compare_stats(s, gold, rate_tol=8e-3, p_min=1e-6, label="trx-ir",
                             keys=["len_aligned", "len_middle_ref", "len_head", "match_run", "first_match", "events_per_read"])
    n_ir = n_iv = 0
    for name, _, _ in rs._records(out + "_aligned_reads.fasta", False):
        if "_RetainedIntron_" in name:
            n_ir += 1
            n_iv += name.split("_RetainedIntron_")[1].split("_")[0].count(";")
    f_d, f_g = n_ir / s["n_aligned"], gold["ir_reads"] / gold["n_aligned"]
    k_d, k_g = n_iv / max(n_ir, 1), gold["ir_intervals"] / max(gold["ir_reads"], 1)
    print("reads with a retained intron: device %.4f reference %.4f; intervals per such read %.3f vs %.3f" % (f_d, f_g, k_d, k_g))
    if abs(f_d - f_g) > 5 * np.sqrt(f_g * (1 - f_g) * (1 / s["n_aligned"] + 1 / gold["n_aligned"])) + 2e-3:
        fails.append("share of IR reads %.4f vs %.4f" % (f_d, f_g))
    if abs(k_d / k_g - 1) > 0.03:
        fails.append("retained intervals per IR read %.3f vs %.3f" % (k_d, k_g))
    assert not fails, "\n".join(fails)


def test_lognormal_lengths_med_sd(ecoli, L):
    """-med / -sd (simulator.py:1285-1295, 1494-1495): log-normal read lengths."""
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=False, seed=5)
    eng.configure(fastq=False, min_len=50, max_len=ecoli.max_chrom, median_len=5000, sd_len=0.4)
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 20000)
    bu = eng.fetch()
    # unaligned: ref ~ lognormal(log(5000), 0.4); the read is the mutated copy (ins ~ del in expectation)
    assert abs(np.median(bu.pieces["ref_req"]) / 5000 - 1) < 0.02
    assert abs(np.std(np.log(bu.pieces["ref_req"].astype(np.float64))) - 0.4) < 0.01
    eng.simulate(L.NS_KIND_ALIGNED, 0, 20000)
    ba = eng.fetch()
    # aligned: total ~ lognormal(log(5000 + 0.08), 0.4) minus/plus independent remainders, then errors (~ -2.8 % net)
    med = np.median(ba.reads["seq_len"])
    assert 4500 < med < 5400, med
    eng.close()


def test_quality_draws_match_model_pmf(ecoli, L):
    """Device qualities per state against the exact truncated-log-normal pmf (model_base_qualities.py:9-20,120-130)."""
    eng, cm, t = pc.make_engine("guppy", ecoli, fastq=True, seed=31)
    eng.simulate(L.NS_KIND_ALIGNED, 0, 20000)
    b = eng.fetch(want_ops=False)
    s = pc.batch_stats(b, ecoli, True)
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 4000)
    pc.batch_stats(eng.fetch(), ecoli, True, s)
    eng.close()
    from nanosim_b200.model import QUAL_STATES
    for key, st in (("qual_ht", "ht"), ("qual_unaligned", "unmapped")):
        pm = t.qual_pmf[QUAL_STATES.index(st)]
        stat, dof, p = pc.chi2_two_sample(s[key], pm * 1e12)
        assert p > 1e-6, (key, stat, dof, p)
    # the aligned middle is a mixture of match / mis / ins states weighted by the simulated base counts
    mix = (t.qual_pmf[QUAL_STATES.index("match")] * (s["aligned_bases"] - s["head_bases"] - s["tail_bases"]))
    assert s["qual_middle"].sum() == s["aligned_bases"] - s["head_bases"] - s["tail_bases"]
    assert s["qual_middle"][:1].sum() == 0 and s["qual_middle"][1:].sum() > 0
    assert abs(np.average(np.arange(94), weights=s["qual_middle"]) - np.average(np.arange(94), weights=mix)) < 1.5


def test_cli_end_to_end_config1(tmp_path, L):
    """BASELINE config 1 through the drop-in command line: file names, formats and read counts of the reference."""
    from nanosim_b200 import simulator
    from nanosim_b200.model import CompiledModel
    ref_path = os.path.join(str(tmp_path), "ecoli5m.fa")
    synth.ecoli5m(ref_path)
    out = os.path.join(str(tmp_path), "sim")
    simulator.main(["genome", "-rg", ref_path, "-c", os.path.join(pc.DATA, pc.MODELS["guppy"]), "-n", "1000", "-o", out,
                    "--seed", "7"])
    s = rs.stats_from_prefix(out, False)
    assert (s["n_aligned"], s["n_unaligned"]) == (898, 102)          # round(1000*8.85/9.85), simulator.py:541
    assert open(out + "_aligned_error_profile").readline() == "Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n"
    r = pc.rates(s)
    assert 0.025 < r["mis"] < 0.036 and 0.019 < r["ins"] < 0.03 and 0.045 < r["del"] < 0.058
    names = [l[1:].strip() for l in open(out + "_unaligned_reads.fasta") if l.startswith(">")]
    assert [int(n.split("_unaligned_")[1].split("_")[0]) for n in names] == list(range(898, 1000))
    out2 = os.path.join(str(tmp_path), "simq")
    simulator.main(["genome", "-rg", ref_path, "-c", os.path.join(pc.DATA, pc.MODELS["dorado"]), "-n", "300", "-o", out2,
                    "--fastq", "--chimeric", "-t", "4"])
    s2 = rs.stats_from_prefix(out2, True)
    assert s2["n_aligned"] + s2["n_unaligned"] == 300 and s2["qual_middle"].sum() > 0


_FETCH_DIGEST = """
import hashlib, os, sys
sys.path[:0] = [%r, %r, %r]
import parity_checks as pc
from nanosim_b200 import _lib as L
from nanosim_b200.reference_fasta import PackedReference
import synth
refs = [PackedReference.from_records(synth.ecoli5m()), PackedReference.from_fasta(os.path.join(%r, "mini_ref.fa"))]
h = hashlib.sha256()
packs = []
for ref in refs:
    eng, _, _ = pc.make_engine("guppy", ref, seed=99, fastq=True)
    packs.append(int(eng.fetch_packs_bases()))
    for kind, n in ((L.NS_KIND_ALIGNED, 1500), (L.NS_KIND_UNALIGNED, 300)):
        eng.simulate(kind, 7, n)
        b = eng.fetch()
        for r in b.reads:
            a, m = int(r["seq_off"]), int(r["seq_len"])
            h.update(b.seq[a:a + m].tobytes())
            h.update(b.qual[a:a + m].tobytes())
    eng.close()
print("DIGEST", h.hexdigest(), packs)
"""


def test_fetch_two_bit_transfer_equals_ascii_transfer():
    """ns_fetch sends the bases over PCIe as 2 bits each and expands them on the host (AVX2 / table) when the reference holds
    nucleotide codes only and the process has CPU cores for it; otherwise as ASCII.  Same seed => same bytes either way:
    NANOSIM_B200_UNPACK_THREADS=0 forces ASCII, =3 forces three expanding threads (the choice is made once per process, hence
    the subprocesses).  References: pure ACGT, and the IUPAC / lower-case mini reference."""
    import subprocess
    from conftest import ROOT
    code = _FETCH_DIGEST % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), GOLDEN)
    out = {}
    for nt in ("0", "3"):
        env = dict(os.environ, NANOSIM_B200_UNPACK_THREADS=nt, PYTHONPATH=ROOT)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
        line = [l for l in r.stdout.splitlines() if l.startswith("DIGEST")][-1].split(None, 2)
        out[nt] = (line[1], line[2])
    assert out["0"][1] == "[0, 0]" and out["3"][1] == "[1, 1]", out       # ASCII / packed on both references
    assert out["0"][0] == out["3"][0], "2-bit transfer and ASCII transfer give different reads"


# ---------------------------------------------------------------------------------------------------------------------
# BASELINE configs 3, 4 and 5 on their named synthetic references (SURVEY.md 8d generators, tests/synth.py), small N
# against the pinned oracle
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_files(prefix, sink, fastq):
    with open(prefix + "_aligned_reads" + (".fastq" if fastq else ".fasta"), "w") as f:
        import nanosim_oracle as no
        f.write(no.format_records(sink.records, fastq))
    with open(prefix + "_aligned_error_profile", "w") as f:
        f.write("Seq_name\tSeq_pos\terror_type\terror_length\tref_base\tseq_base\n")
        f.writelines(r + "\n" for r in sink.error_rows)
    return rs.stats_from_prefix(prefix, fastq)


def test_config3_transcriptome_200k_transcripts_vs_oracle(L, tmp_path):
    """BASELINE config 3: transcriptome directRNA, dRNA_Bham1_guppy model, FASTA, --no_model_ir, on the 200k-transcript
    synthetic reference with its expression profile (simulator.py:1043-1263).  Aligned reads: length laws, error rates, the
    aligned share of the chosen transcript, the lengths of the chosen transcripts.  Unaligned reads: a uniformly chosen
    transcript longer than the read (:1695-1703) -- on the device one draw among the records sorted by length."""
    import random
    import nanosim_oracle as no
    from conftest import oracle_model
    from nanosim_b200.reference_fasta import PackedReference
    names, lengths, bases, tpm = synth.config3_transcriptome()
    keys = [n.split(".")[0] for n in names]
    offs = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    ref = PackedReference(keys, bases, offs)
    N = 500
    eng, cm, t = pc.make_trx_engine(ref, np.arange(len(keys), dtype=np.uint32), tpm, None, fastq=False, seed=303, kde2d_sample=N)
    s_dev = rs.empty()
    eng.simulate(L.NS_KIND_ALIGNED, 0, 60000)
    b = eng.fetch(want_ops=True)
    assert pc.check_edit_scripts(b, ref, False, max_reads=400) > 0
    pc.meta_stats(b, s_dev)
    pc.merge_op_stats(s_dev, eng.op_stats())
    tl_dev = ref.lengths[b.pieces["chrom"]]
    frac_dev = b.pieces["ref_len"] / tl_dev
    eng.simulate(L.NS_KIND_UNALIGNED, 0, 40000)
    bu = eng.fetch()
    pc.meta_stats(bu, s_dev)
    tlu_dev = ref.lengths[bu.pieces["chrom"]]
    assert (bu.pieces["ref_len"] < tlu_dev).all() and (bu.pieces["pos"].astype(np.int64) + bu.pieces["ref_len"] <= tlu_dev).all()
    eng.close()
    seqs = [bases[int(offs[i]):int(offs[i + 1])].tobytes().decode() for i in range(len(keys))]
    oref = no.OracleTrxReference(list(zip(keys, seqs)), dict(zip(keys, tpm.tolist())))
    m = oracle_model(cm, tmp_path, fastq=False)
    s_or = rs.empty()
    tl_or, frac_or, tlu_or = [], [], []
    index = {k: i for i, k in enumerate(keys)}
    for rep in range(2):
        random.seed(700 + rep)
        np.random.seed(700 + rep)
        sink = no.ReadSink()
        no.simulation_aligned_transcriptome(oref, m, sink, None, "guppy", N, False, False, False, False, False)
        rs.merge(s_or, _oracle_files(os.path.join(str(tmp_path), "o3_%d" % rep), sink, False))
        for name, seq, q in sink.records:
            i = index[name.split("_")[0]]
            tl_or.append(lengths[i])
            frac_or.append(int(name.rsplit("_", 4)[3]) / lengths[i])
    random.seed(710)
    np.random.seed(710)
    sink_u = no.ReadSink()
    no.simulation_unaligned_transcriptome(oref, m, sink_u, 50, oref.max_chrom, False, 1200)
    for name, seq, q in sink_u.records:
        tlu_or.append(lengths[index[name.split("_")[0]]])
        s_or["len_unaligned"][rs._bin(rs.LEN_EDGES, len(seq))] += 1
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.06, p_min=1e-5, label="config3",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match", "len_unaligned"])
    ledges = np.unique(np.round(np.logspace(np.log10(300), np.log10(20001), 25)))
    for label, x, y, edges in (("length of the chosen transcript (aligned)", tl_dev, tl_or, ledges),
                               ("length of the chosen transcript (unaligned)", tlu_dev, tlu_or, ledges),
                               ("aligned share of the transcript", frac_dev, frac_or, np.linspace(0, 1.0001, 21))):
        st, dof, p = pc.chi2_two_sample(np.histogram(x, edges)[0], np.histogram(y, edges)[0])
        print("config3 %s: chi2 %.1f dof %d p %.3g" % (label, st, dof, p))
        if p < 1e-5:
            fails.append("config3 %s: chi2 %.1f dof %d p %.3g" % (label, st, dof, p))
    assert not fails, "\n".join(fails)


def test_config4_metagenome_50_species_vs_oracle(L, tmp_path):
    """BASELINE config 4: metagenome, ERR3152364_Even model, FASTQ --chimeric, 50 species x 1-3 circular chromosomes, Even
    abundance (simulator.py:814-1040, assign_species :758-811): device vs the pinned oracle on the same reference, and the
    species base shares against the abundance the quotas enforce."""
    import random
    import nanosim_oracle as no
    from conftest import oracle_model
    from nanosim_b200.reference_fasta import MetaReference
    genomes = synth.config4_metagenome()
    ref = MetaReference.from_genomes(genomes)
    abun = [100.0 / len(ref.species)] * len(ref.species)
    eng, cm, t = pc.make_meta_engine(ref, abun, fastq=True, chimeric=True, seed=404)
    s_dev = rs.empty()
    fr = np.zeros(len(ref.species))
    for k in range(3):
        eng.simulate(L.NS_KIND_ALIGNED, k * 12000, 12000)
        b = eng.fetch(want_ops=(k == 0))
        if k == 0:
            assert pc.check_edit_scripts(b, ref, True, max_reads=300) > 0
            b.ops = None                                  # event histograms come from the device (ns_op_stats)
        pc.batch_stats(b, ref, True, s_dev)               # lengths, strands, quality histograms
        pc.merge_op_stats(s_dev, eng.op_stats())
        fr += _species_base_fractions(b, ref, L) / 3
    eng.close()
    print("config4 species base shares: min %.4f max %.4f (target %.4f)" % (fr.min(), fr.max(), 1.0 / len(ref.species)))
    assert np.abs(fr - 1.0 / len(ref.species)).max() < 2e-3             # quota fill: every species gets its share of the bases
    oref = no.OracleMetaReference({MetaReference.species_key(sp): [(k2, a.tobytes().decode()) for k2, a in recs] for sp, recs in genomes})
    m = oracle_model(cm, tmp_path, fastq=True, chimeric=True, mode="metagenome")
    oabun = {sp: a for sp, a in zip(ref.species, abun)}
    infl = {sp: no.inflate_abun(oabun, sp, m.abun_inflation) for sp in oabun}
    random.seed(44)
    np.random.seed(44)
    sink = no.ReadSink()
    no.simulation_aligned_metagenome(oref, m, sink, oabun, infl, 50, max(oref.max_chrom.values()), None, True, 500, False, True)
    s_or = _oracle_files(os.path.join(str(tmp_path), "o4"), sink, True)
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.05, p_min=1e-5, label="config4",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    for k in ("qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        print("config4", k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-5:
            fails.append("config4 %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    fc_d, fc_o = s_dev["n_chimeric"] / s_dev["n_aligned"], s_or["n_chimeric"] / s_or["n_aligned"]
    assert abs(fc_d - fc_o) < 0.035, (fc_d, fc_o)
    assert not fails, "\n".join(fails)


def test_config5_dorado_hp_chimeric_on_3gb_reference_vs_oracle(L, tmp_path):
    """BASELINE config 5 (and the reference of config 2): genome, dorado kit-v14 model, FASTQ -hp -k 6 --chimeric on the 3.09 Gb
    synthetic reference (24 chromosomes with hg38 lengths).  Device vs the pinned oracle: lengths, error rates after the
    homopolymer filter (simulator.py:1920-1947), run lengths after mutate_homo (:618-705), qualities; plus the bit-exact
    script check on chromosomes of hundreds of Mb (offsets beyond 2^31)."""
    import torch
    from nanosim_b200.reference_fasta import PackedReference
    rng = np.random.default_rng(1)
    lens = synth.HG38_LENGTHS
    g = torch.Generator(device="cuda:0")
    g.manual_seed(1)
    lut = torch.tensor([65, 67, 71, 84], dtype=torch.uint8, device="cuda:0")
    total = sum(lens)
    dev = torch.empty(total, dtype=torch.uint8, device="cuda:0")
    for s0 in range(0, total, 1 << 28):
        e0 = min(total, s0 + (1 << 28))
        dev[s0:e0] = lut[torch.randint(0, 4, (e0 - s0,), generator=g, device="cuda:0", dtype=torch.uint8).long()]
    bases = dev.cpu().numpy()
    del dev
    torch.cuda.empty_cache()
    ref = PackedReference(list(synth.HG38_NAMES), bases, np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64))
    eng, cm, t = pc.make_engine("dorado", ref, fastq=True, chimeric=True, kmer_bias=6, seed=505)
    s_dev = rs.empty()
    eng.simulate(L.NS_KIND_ALIGNED, 0, 3000)
    b = eng.fetch(want_ops=True)
    assert pc.check_edit_scripts(b, ref, True, max_reads=150) > 0
    assert (b.pieces["chrom"] > 10).any() and int((ref.offsets[b.pieces["chrom"]].astype(np.int64) + b.pieces["pos"]).max()) > 2 ** 31
    pc.batch_stats(b, ref, True, s_dev)
    eng.close()
    recs = [(n, bases[int(ref.offsets[i]):int(ref.offsets[i + 1])].tobytes().decode()) for i, n in enumerate(ref.names)]
    s_or = pc.oracle_stats(cm, recs, 160, 0, True, chimeric=True, tmpdir=str(tmp_path), kmer_bias=6)
    fails = pc.compare_stats(s_dev, s_or, rate_tol=0.08, p_min=1e-5, label="config5",
                             keys=["len_aligned", "len_middle_ref", "len_head", "len_tail", "match_run", "first_match"])
    for k in ("hp_runs", "qual_middle", "qual_ht"):
        st, dof, p = pc.chi2_two_sample(s_dev[k], s_or[k])
        print("config5", k, "chi2 %.1f dof %d p %.3g" % (st, dof, p))
        if p < 1e-5:
            fails.append("config5 %s chi2 %.1f dof %d p %.3g" % (k, st, dof, p))
    rd = (s_dev["aligned_bases"] - s_dev["head_bases"] - s_dev["tail_bases"]) / s_dev["ref_bases"]
    ro = (s_or["aligned_bases"] - s_or["head_bases"] - s_or["tail_bases"]) / s_or["ref_bases"]
    print("config5 middle bases per reference base: device %.5f oracle %.5f" % (rd, ro))
    assert abs(rd / ro - 1) < 3e-3, (rd, ro)
    assert not fails, "\n".join(fails)
