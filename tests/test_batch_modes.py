"""Sized and sync-free batches (run on an H100: ``pytest -m gpu``).

The first batch of a kind is sized: the host reads the totals mid-pipeline and grows the buffers.  A later batch that fits
them is submitted in one go and checks the capacities on the device (DESIGN §3).  Both modes must compute the same batch.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN

import parity_checks as pc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mini_ref():
    from nanosim_b200.reference_fasta import PackedReference
    return PackedReference.from_fasta(os.path.join(GOLDEN, "mini_ref.fa"))


@pytest.fixture(scope="module")
def trx_ref():
    from nanosim_b200.reference_fasta import PackedReference, read_expression, read_polya_list
    T = os.path.join(GOLDEN, "trx")
    ref = PackedReference.from_fasta(os.path.join(T, "transcripts.fa"))
    chrom, w = read_expression(os.path.join(T, "expression.tsv"), ref)
    return ref, chrom, w, read_polya_list(os.path.join(T, "polya.txt"), ref)


def _piece_scripts(b):
    """Every piece's emitted script and event script."""
    return [(b.ops[int(p["op_off"]):int(p["op_off"]) + int(p["n_ops"])].tobytes(),
             b.ops[int(p["ev_off"]):int(p["ev_off"]) + int(p["ev_n_ops"])].tobytes()) for p in b.pieces]


@pytest.mark.parametrize("mode", ["genome", "transcriptome"])
def test_sync_free_batch_equals_sized_batch(mode, mini_ref, trx_ref):
    """The same batch simulated twice in one context, sized and then sync-free, gives the same bytes, records, scripts
    and totals."""
    from nanosim_b200 import _lib as L

    if mode == "genome":
        eng, _, _ = pc.make_engine("guppy", mini_ref, fastq=True, seed=5)
    else:
        ref, chrom, w, polya = trx_ref
        eng, _, _ = pc.make_trx_engine(ref, chrom, w, polya, fastq=True, seed=5)
    for kind in (L.NS_KIND_ALIGNED, L.NS_KIND_UNALIGNED):
        (sized, a), (sync_free, b) = [(eng.simulate(kind, 17, 2000), eng.fetch(want_ops=True)) for _ in range(2)]
        for f in ("seq_bytes", "n_ops", "total_bases", "n_reads", "n_pieces"):
            assert getattr(sized, f) == getattr(sync_free, f), f
        for f in ("seq", "qual", "reads"):
            assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f
        # unaligned reads that are drawn again take their script's slot from a pool with an atomic: op_off / ev_off vary
        # from run to run, the scripts they locate do not
        for f in L.PIECE_DTYPE.names:
            assert f in ("op_off", "ev_off") or np.array_equal(a.pieces[f], b.pieces[f]), f
        assert _piece_scripts(a) == _piece_scripts(b)
        # the second batch really ran sync-free: a capacity check, the replay of the reads whose script overflowed its slot
        # (always submitted, 2 launches) and one publish of the totals, where a sized batch publishes its totals twice and
        # replays only when there are such reads
        flagged = bool((a.reads["flags"] & 1).any())
        assert sync_free.n_launches == sized.n_launches + (0 if flagged else 2)
    eng.close()
