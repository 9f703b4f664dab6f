"""The device's random draw primitives against their own definitions.

tests/draw_harness.cu runs the library's draw functions (device_common.cuh, emit_kernel.cuh, qual_table.h) over whole
input spaces or over every boundary word; each result is compared here with a float64 or exact-integer reference of the
same draw.  The integer primitives run on the host path too (no GPU needed); on the device they must give the same
results, which they do when both equal the reference.  What is held, and the residual biases it pins:

  * Philox4x32-10 against the Random123 known-answer vectors, -10 and -7 against a NumPy restatement of the round;
  * both Walker alias samplers per word against the table's definition, and the realised counts of all 2^32 words
    against the closed form (within n 2^-32 of the float64 pmf);
  * the quality tables: every 24-bit draw, counts equal to the 24-bit pmf exactly;
  * substitution offsets 1 : 2 : 3 as 5462 : 5461 : 5461 of 4^7 (bias 4^-7);
  * the three-way draws of event bases and IUPAC codes D V H B as 21846 : 21845 : 21845 of 2^16 (bias 2^-15);
  * the Box-Muller factors within 2 ulp of float64 and the realised normal CDF within 1e-6 of Phi.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import DATA, MODEL_FILES
from parity_checks import _IUPAC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nanosim_b200", "csrc")
HARNESS = os.path.join(ROOT, "tests", "draw_harness.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]     # as __graft_entry__.build

M32 = 0xFFFFFFFF
ST_EMIT_B, ST_IUPAC = 6, 7                   # device_common.cuh stream purposes
ACTG = "ACTG"                                # base index order of the device (A 0, C 1, T 2, G 3)


def _build(out_dir, host_only):
    so = os.path.join(str(out_dir), "draw_harness_host.so" if host_only else "draw_harness.so")
    cmd = [NVCC] + FLAGS + ["-shared", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
                            "-o", so, HARNESS] + (["-DDRAW_HARNESS_HOST_ONLY"] if host_only else [])
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout + r.stderr
    lib = ctypes.CDLL(so)
    for name in ("dh_philox", "dh_sub_offsets", "dh_add_fields_mod4", "dh_event_base_all", "dh_event_bases", "dh_iupac16_all",
                 "dh_converted_ref_base", "dh_build_qlut", "dh_qual_all", "dh_alias", "dh_alias_all_words", "dh_normal_factors"):
        getattr(lib, name).restype = ctypes.c_int
    return lib


class Harness:
    """One side of the harness: numpy arrays in and out; on the device side they go through torch CUDA tensors."""

    def __init__(self, lib, dev):
        self.lib, self.dev = lib, dev

    def _in(self, a):
        a = np.ascontiguousarray(a)
        if not self.dev:
            return a
        import torch

        return torch.from_numpy(a.view({4: np.int32, 8: np.int64}.get(a.itemsize, a.dtype))).cuda()

    def _out(self, n, dtype):
        if not self.dev:
            return np.zeros(n, dtype=dtype)
        import torch

        return torch.zeros(n, dtype={1: torch.uint8, 4: torch.int32}[np.dtype(dtype).itemsize], device="cuda")

    @staticmethod
    def _p(x):
        return ctypes.c_void_p(x.ctypes.data if isinstance(x, np.ndarray) else x.data_ptr())

    @staticmethod
    def _np(x, dtype):
        return x if isinstance(x, np.ndarray) else x.cpu().numpy().view(dtype)

    def call(self, name, *args):
        err = getattr(self.lib, name)(*args)
        assert err == 0, "%s: cudaError %d" % (name, err)

    def philox(self, rounds, ctr, key):
        c, k, o = self._in(ctr.astype(np.uint32)), self._in(key.astype(np.uint32)), self._out(4 * len(ctr), np.uint32)
        self.call("dh_philox", ctypes.c_int(self.dev), ctypes.c_int(rounds), self._p(c), self._p(k), self._p(o), ctypes.c_uint64(len(ctr)))
        return self._np(o, np.uint32).reshape(-1, 4)

    def sub_offsets(self, x):
        xi, o = self._in(x.astype(np.uint32)), self._out(len(x), np.uint32)
        self.call("dh_sub_offsets", ctypes.c_int(self.dev), self._p(xi), self._p(o), ctypes.c_uint64(len(x)))
        return self._np(o, np.uint32)

    def add_fields_mod4(self, a, b):
        ai, bi, o = self._in(a.astype(np.uint32)), self._in(b.astype(np.uint32)), self._out(len(a), np.uint32)
        self.call("dh_add_fields_mod4", ctypes.c_int(self.dev), self._p(ai), self._p(bi), self._p(o), ctypes.c_uint64(len(a)))
        return self._np(o, np.uint32)

    def event_base_all(self):
        o = self._out((1 << 18) + (1 << 16), np.uint8)
        self.call("dh_event_base_all", ctypes.c_int(self.dev), self._p(o))
        return self._np(o, np.uint8)

    def event_bases(self, seed, rid, piece, event, mis, orig):
        oi, o = self._in(orig.astype(np.uint8)), self._out(len(orig), np.uint8)
        self.call("dh_event_bases", ctypes.c_int(self.dev), ctypes.c_uint64(seed), ctypes.c_uint64(rid), ctypes.c_uint32(piece),
                  ctypes.c_uint32(event), ctypes.c_uint32(int(mis)), self._p(oi), self._p(o), ctypes.c_uint64(len(orig)))
        return self._np(o, np.uint8)

    def iupac16_all(self):
        o = self._out(1 << 24, np.uint8)
        self.call("dh_iupac16_all", ctypes.c_int(self.dev), self._p(o))
        return self._np(o, np.uint8).reshape(256, 1 << 16)

    def converted_ref_base(self, seed, rid, piece, c, off):
        ci, fi, o = self._in(c.astype(np.uint8)), self._in(off.astype(np.uint32)), self._out(len(c), np.uint8)
        self.call("dh_converted_ref_base", ctypes.c_int(self.dev), ctypes.c_uint64(seed), ctypes.c_uint64(rid), ctypes.c_uint32(piece),
                  self._p(ci), self._p(fi), self._p(o), ctypes.c_uint64(len(c)))
        return self._np(o, np.uint8)

    def qual_all(self, lut):
        li, o = self._in(lut), self._out(5 << 24, np.uint8)
        self.call("dh_qual_all", ctypes.c_int(self.dev), self._p(li), self._p(o))
        return self._np(o, np.uint8).reshape(5, 1 << 24)


@pytest.fixture(scope="session")
def host_harness(tmp_path_factory):
    return Harness(_build(tmp_path_factory.mktemp("draw_harness_host"), host_only=True), 0)


@pytest.fixture(scope="session")
def device_lib(tmp_path_factory):
    import torch

    if not torch.cuda.is_available():
        pytest.fail("the device draw tests need a CUDA device")
    return _build(tmp_path_factory.mktemp("draw_harness"), host_only=False)


@pytest.fixture(params=["host", pytest.param("device", marks=pytest.mark.gpu)])
def harness(request):
    if request.param == "host":
        return request.getfixturevalue("host_harness")
    return Harness(request.getfixturevalue("device_lib"), 1)


# ---------------------------------------------------------------------------------------------------------------------
# Philox4x32
# ---------------------------------------------------------------------------------------------------------------------
def philox_ref(ctr, key, rounds):
    """Philox4x32-R (Salmon et al., SC'11) in uint64 arithmetic: ctr [n,4], key [n,2] -> [n,4]."""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = key[:, 0].astype(np.uint64), key[:, 1].astype(np.uint64)
    m = np.uint64(M32)
    for _ in range(rounds):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & m, p1 & m, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & m, p0 & m]
        k0 = (k0 + np.uint64(0x9E3779B9)) & m
        k1 = (k1 + np.uint64(0xBB67AE85)) & m
    return np.stack(c, axis=1).astype(np.uint32)


def test_philox10_known_answers(harness):
    """The Random123 known-answer vectors of Philox4x32-10 (kat_vectors: zero, all-ones, digits of pi)."""
    ctr = np.array([[0, 0, 0, 0], [M32] * 4, [0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]], dtype=np.uint32)
    key = np.array([[0, 0], [M32, M32], [0xa4093822, 0x299f31d0]], dtype=np.uint32)
    want = np.array([[0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8], [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd],
                     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]], dtype=np.uint32)
    np.testing.assert_array_equal(harness.philox(10, ctr, key), want)
    np.testing.assert_array_equal(philox_ref(ctr, key, 10), want)


@pytest.mark.parametrize("rounds", [10, 7])
def test_philox_matches_restatement(harness, rounds):
    """2^20 random (counter, key) pairs plus the carry edges: every word 0, 0xfffffffe or 0xffffffff in every
    combination, with the same keys."""
    rng = np.random.default_rng(rounds)
    n = 1 << 20
    ctr = rng.integers(0, 1 << 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    key = rng.integers(0, 1 << 32, size=(n, 2), dtype=np.uint64).astype(np.uint32)
    edge = np.array(np.meshgrid(*[[0, 0xfffffffe, M32]] * 6, indexing="ij"), dtype=np.uint64).reshape(6, -1).T.astype(np.uint32)
    ctr = np.concatenate([ctr, edge[:, :4]])
    key = np.concatenate([key, edge[:, 4:]])
    got = harness.philox(rounds, ctr, key)
    want = philox_ref(ctr, key, rounds)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, "first mismatch: ctr %s key %s: %s != %s" % (ctr[bad[0]], key[bad[0]], got[bad[0]], want[bad[0]])


# ---------------------------------------------------------------------------------------------------------------------
# substitutions of the emit kernel
# ---------------------------------------------------------------------------------------------------------------------
def _fields(w):
    """[n] uint32 -> [n, 16] 2-bit fields."""
    return (w[:, None].astype(np.int64) >> (2 * np.arange(16))) & 3


def _words(f):
    """[n, 16] fields -> [n] uint32."""
    return (f.astype(np.uint64) << (2 * np.arange(16, dtype=np.uint64))).sum(axis=1).astype(np.uint32)


def test_sub_offsets_exact_enumeration(harness):
    """Per field position: all 4^7 values of that field's seven 2-bit draws, the other fields random.  Field i of the
    result is the first non-zero draw of field i (1 if all seven are zero): never 0, and 1 : 2 : 3 come out exactly
    5462 : 5461 : 5461 times (bias 4^-7)."""
    rng = np.random.default_rng(7)
    combos = (np.arange(4 ** 7)[:, None] >> (2 * np.arange(7))) & 3               # [16384, 7]: draws X1..X7 of one field
    fields = rng.integers(0, 4, size=(16, 4 ** 7, 7, 16), dtype=np.int8)
    for f in range(16):
        fields[f, :, :, f] = combos
    fields = fields.reshape(-1, 7, 16)
    x = np.stack([_words(fields[:, d, :]) for d in range(7)], axis=1)
    got = _fields(harness.sub_offsets(x))
    nz = fields != 0
    first = np.argmax(nz, axis=1)                                                 # [n, 16]
    want = np.where(nz.any(axis=1), np.take_along_axis(fields, first[:, None, :], axis=1)[:, 0, :], 1)
    np.testing.assert_array_equal(got, want)                                      # field i depends on field i only
    assert (got != 0).all()
    got = got.reshape(16, 4 ** 7, 16)
    for f in range(16):
        counts = np.bincount(got[f, :, f], minlength=4)
        assert counts.tolist() == [0, 5462, 5461, 5461], (f, counts)


def test_add_fields_mod4(harness):
    """Every field position with all 4 x 4 values, other fields random, plus 2^16 random pairs: (a + b) mod 4 per field."""
    rng = np.random.default_rng(4)
    a = rng.integers(0, 4, size=(16, 16, 16))
    b = rng.integers(0, 4, size=(16, 16, 16))
    for f in range(16):
        a[f, :, f] = np.arange(16) >> 2
        b[f, :, f] = np.arange(16) & 3
    a, b = _words(a.reshape(-1, 16)), _words(b.reshape(-1, 16))
    a = np.concatenate([a, rng.integers(0, 1 << 32, size=1 << 16, dtype=np.uint64).astype(np.uint32)])
    b = np.concatenate([b, rng.integers(0, 1 << 32, size=1 << 16, dtype=np.uint64).astype(np.uint32)])
    np.testing.assert_array_equal(_fields(harness.add_fields_mod4(a, b)), (_fields(a) + _fields(b)) & 3)


# ---------------------------------------------------------------------------------------------------------------------
# three-way draws: bases of events the homopolymer pass rewrites, IUPAC codes
# ---------------------------------------------------------------------------------------------------------------------
def three_way_ref(h):
    """Index 0, 1, 2 of a pick among three from 16 uniform bits: 21846 : 21845 : 21845."""
    return (np.asarray(h, dtype=np.int64) * 3) >> 16


def test_event_base_three_way_counts(harness):
    """Every 16-bit draw h for each original base: a substituted base is never the original, and the three others come
    out at most 1 apart in 2^16 (21846 : 21845 : 21845, relative bias 2^-15); an inserted base is exactly uniform."""
    out = harness.event_base_all()
    h = np.arange(1 << 16)
    for orig in range(4):
        got = out[(orig << 16) + h].astype(np.int64)
        counts = np.bincount(got, minlength=4)
        others = [counts[(orig + k) & 3] for k in (1, 2, 3)]
        assert counts[orig] == 0 and max(others) - min(others) <= 1, \
            "MIS from %s: counts of A C T G = %s" % (ACTG[orig], counts.tolist())
        np.testing.assert_array_equal(got, (orig + 1 + three_way_ref(h)) & 3)
    ins = out[(1 << 18) + h].astype(np.int64)
    assert np.bincount(ins, minlength=4).tolist() == [1 << 14] * 4
    np.testing.assert_array_equal(ins, h & 3)


def _event_draws(seed, rid, piece, event, n):
    """16-bit draw of base t of an event: half t % 2 of word (t >> 1) % 4 of Philox-7 block (event << 9) + (t >> 3) on
    stream ST_EMIT_B of the piece."""
    t = np.arange(n, dtype=np.uint64)
    ctr = np.stack([np.full(n, rid & M32), np.full(n, rid >> 32), np.full(n, (ST_EMIT_B << 28) | piece),
                    (np.uint64(event) << np.uint64(9)) + (t >> np.uint64(3))], axis=1).astype(np.uint32)
    key = np.tile(np.array([seed & M32, seed >> 32], dtype=np.uint32), (n, 1))
    blk = philox_ref(ctr, key, 7)
    word = blk[np.arange(n), ((t >> np.uint64(1)) & np.uint64(3)).astype(np.int64)].astype(np.int64)
    return (word >> (16 * (t & np.uint64(1)).astype(np.int64))) & 0xFFFF


@pytest.mark.parametrize("seed,rid,piece,event", [(0, 0, 0, 0), (0x0123456789abcdef, (7 << 32) | 12345, 3, 4095),
                                                   (2 ** 64 - 1, 2 ** 40 + 1, 0x07ffffff, (1 << 23) - 1)])
def test_event_bases_follow_block_layout(harness, seed, rid, piece, event):
    """The 4096 bases an event can have, drawn through event_base_block / event_draw, against the layout restated on
    Philox-7; the error-profile mirror in records.py gives the same bases."""
    from nanosim_b200.records import event_bases_hp

    n = 4096
    h = _event_draws(seed, rid, piece, event, n)
    orig = np.random.default_rng(event).integers(0, 4, size=n)
    for mis in (True, False):
        got = harness.event_bases(seed, rid, piece, event, mis, orig).astype(np.int64)
        want = (orig + 1 + three_way_ref(h)) & 3 if mis else h & 3
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(event_bases_hp(seed, rid, piece, event, n, mis, orig if mis else None), want)


def _iupac_ref():
    """[256, 2^16] expected result of resolving byte c with 16 bits h: members in case_convert's list order; two- and
    four-member codes by bits [5:4] of h, three-member codes by the three-way pick; every other byte unchanged."""
    h = np.arange(1 << 16)
    out = np.tile(np.arange(256, dtype=np.uint8)[:, None], (1, 1 << 16))
    for code, members in _IUPAC.items():
        m = np.frombuffer(members.encode(), dtype=np.uint8)
        k = three_way_ref(h) if len(m) == 3 else (h >> 4) & (len(m) - 1)
        out[ord(code)] = m[k]
    return out


def test_iupac_resolution_every_draw(harness):
    """Every byte with every 16-bit draw.  Two- and four-member codes are exactly uniform, D V H B at most 1 apart in
    2^16; every byte that is not an upper-case IUPAC code comes back unchanged."""
    got = harness.iupac16_all()
    want = _iupac_ref()
    for code, members in _IUPAC.items():
        counts = np.bincount(got[ord(code)], minlength=256)
        c = [int(counts[ord(b)]) for b in members]
        assert sum(c) == 1 << 16 and max(c) - min(c) <= (1 if len(members) == 3 else 0), \
            "%s -> %s: counts %s" % (code, members, c)
    bad = np.argwhere(got != want)
    assert len(bad) == 0, "byte %r h=%d: %r != %r" % (chr(bad[0][0]), bad[0][1], chr(got[tuple(bad[0])]), chr(want[tuple(bad[0])]))


def test_converted_ref_base_follows_layout(harness):
    """converted_ref_base for every byte, both cases, at offsets 0..63 and far ones: upper-cased, ACGT kept, IUPAC codes
    resolved with the 16 bits of half f % 2 of word (f >> 1) % 4 of Philox-7 block f >> 3 on stream ST_IUPAC."""
    seed, rid, piece = 0x5eed0000cafe, (3 << 32) | 99, 5
    off = np.concatenate([np.arange(64), [1 << 20, (1 << 32) - 1]]).astype(np.uint64)
    c = np.repeat(np.arange(256), len(off)).astype(np.uint8)
    f = np.tile(off, 256)
    got = harness.converted_ref_base(seed, rid, piece, c, f.astype(np.uint32))
    n = len(c)
    ctr = np.stack([np.full(n, rid & M32), np.full(n, rid >> 32), np.full(n, (ST_IUPAC << 28) | piece), f >> np.uint64(3)],
                   axis=1).astype(np.uint32)
    blk = philox_ref(ctr, np.tile(np.array([seed & M32, seed >> 32], dtype=np.uint32), (n, 1)), 7)
    word = blk[np.arange(n), ((f >> np.uint64(1)) & np.uint64(3)).astype(np.int64)].astype(np.int64)
    h = (word >> (16 * (f & np.uint64(1)).astype(np.int64))) & 0xFFFF
    upper = np.where((c >= ord("a")) & (c <= ord("z")), c - 32, c).astype(np.int64)
    want = _iupac_ref()[upper, h]
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, "byte %r at %d: %r != %r" % (chr(c[bad[0]]), f[bad[0]], chr(got[bad[0]]), chr(want[bad[0]]))


# ---------------------------------------------------------------------------------------------------------------------
# base qualities
# ---------------------------------------------------------------------------------------------------------------------
_QUAL_MODELS = ["guppy", "dorado", "drna"]


def _tables(tag, **kw):
    from nanosim_b200.model import CompiledModel, DeviceTables

    return DeviceTables(CompiledModel.load(os.path.join(DATA, MODEL_FILES[tag])), **kw)


@pytest.mark.parametrize("tag", _QUAL_MODELS)
def test_quality_tables_realise_24bit_pmf(harness, host_harness, tag):
    """All 2^24 draws (11-bit slot, 13-bit threshold) of each of the 5 quality states through build_qlut's table and
    qual_pick: the counts are exactly the 24-bit masses diff(round(cdf / 2^8)), which are within 2^-24 + 2^-32 of the
    float64 pmf; no character outside '"' .. '~' (q 1 .. 93)."""
    t = _tables(tag, fastq=True)
    lut = np.zeros(5 * 2048, dtype=np.uint32)
    host_harness.call("dh_build_qlut", Harness._p(np.ascontiguousarray(t.qual_cdf)), Harness._p(lut))
    got = harness.qual_all(lut)
    for s in range(5):
        counts = np.bincount(got[s], minlength=256).astype(np.int64)
        c24 = np.maximum.accumulate(np.minimum((t.qual_cdf[s].astype(np.int64) + 128) >> 8, 1 << 24))
        c24[-1] = 1 << 24
        mass = np.diff(np.concatenate([[0], c24]))
        assert counts[:34].sum() == 0 and counts[127:].sum() == 0, (s, np.nonzero(counts)[0])
        np.testing.assert_array_equal(counts[33:127], mass, err_msg="state %d" % s)
        assert np.abs(mass / 2.0 ** 24 - t.qual_pmf[s]).max() <= 2.0 ** -24 + 2.0 ** -32


# ---------------------------------------------------------------------------------------------------------------------
# Walker alias tables
# ---------------------------------------------------------------------------------------------------------------------
_ALIAS_BUILDS = {"guppy": ("guppy", {}), "dorado": ("dorado", {}), "even_meta": ("even", {"mode": "metagenome"}),
                 "drna_trx": ("drna", {"mode": "transcriptome"}), "dorado_hp": ("dorado", {"homopolymer": True})}


def _slot_bounds(n, prob):
    """Per slot j of an n-slot table: first word, one past the last word, and the first word whose frac reaches
    prob[j] (the words of slot j are those with (r n) >> 32 == j; their frac = r n mod 2^32 rises in steps of n)."""
    j = np.arange(n, dtype=np.int64)
    lo = -((-(j << 32)) // n)
    hi = -((-((j + 1) << 32)) // n)
    cut = np.where(prob.astype(np.int64) == M32, hi, np.clip(-((-((j << 32) + prob.astype(np.int64))) // n), lo, hi))
    return lo, hi, cut


def alias_exact_counts(prob, alias):
    """How many of the 2^32 words draw each outcome of the table, in exact integers."""
    n = len(prob)
    lo, hi, cut = _slot_bounds(n, prob)
    counts = np.bincount(np.arange(n), weights=cut - lo, minlength=n).astype(np.int64)
    counts += np.bincount(alias.astype(np.int64), weights=hi - cut, minlength=n).astype(np.int64)
    return counts


def _alias_tables(build):
    tag, kw = _ALIAS_BUILDS[build]
    t = _tables(tag, **kw)
    return t, [(int(o), int(n)) for o, n in t.alias_desc]


@pytest.mark.parametrize("build", sorted(_ALIAS_BUILDS))
def test_alias_closed_form_matches_pmf(build):
    """The exact counts every table realises over all 2^32 words agree with the float64 pmf it was built from within
    n 2^-32 per outcome (the device realises these counts: test_alias_all_words_realise_closed_form)."""
    t, desc = _alias_tables(build)
    for k, (off, n) in enumerate(desc):
        counts = alias_exact_counts(t.alias_prob[off:off + n], t.alias_idx[off:off + n])
        assert counts.sum() == 1 << 32
        pmf = np.asarray(t.pmfs[k], dtype=np.float64)
        err = np.abs(counts / 2.0 ** 32 - pmf / pmf.sum()).max()
        assert err <= n * 2.0 ** -32, (k, n, err)


def _alias_device(t):
    import torch

    inter = np.stack([t.alias_prob, t.alias_idx], axis=1).astype(np.uint32)
    return torch.from_numpy(inter.view(np.int32)).cuda(), np.ascontiguousarray(t.alias_desc[:, 0]), np.ascontiguousarray(t.alias_desc[:, 1])


@pytest.mark.gpu
@pytest.mark.parametrize("build", sorted(_ALIAS_BUILDS))
def test_alias_draws_match_definition(device_lib, build):
    """alias_draw and alias_draw_s (table directory in shared memory, as plan_kernel calls it) on every table: for every
    slot its first and last word and the words either side of the acceptance cut, plus 2^24 random words, against
    j = (r n) >> 32, frac = r n mod 2^32, frac < prob[j] or prob[j] == 0xffffffff ? j : alias[j] in int64."""
    import torch

    t, desc = _alias_tables(build)
    alias, tab_off, tab_n = _alias_device(t)
    prob_d = torch.from_numpy(t.alias_prob.astype(np.int64)).cuda()
    ali_d = torch.from_numpy(t.alias_idx.astype(np.int64)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(len(desc))
    for k, (off, n) in enumerate(desc):
        lo, hi, cut = _slot_bounds(n, t.alias_prob[off:off + n])
        edge = np.concatenate([lo, hi - 1, cut - 1, np.minimum(cut, hi - 1)])
        edge = torch.from_numpy(np.clip(edge, 0, M32)).cuda()
        rnd = torch.randint(0, 1 << 32, (1 << 24,), device="cuda", generator=gen, dtype=torch.int64)
        r = torch.cat([edge, rnd])
        r32 = (r - ((r >> 31) << 32)).to(torch.int32)                            # the same 32 bits
        tt = torch.full_like(r32, k)
        plain, shared = torch.empty_like(r32), torch.empty_like(r32)
        err = device_lib.dh_alias(Harness._p(alias), Harness._p(tab_off), Harness._p(tab_n), ctypes.c_uint32(len(desc)),
                                  Harness._p(tt), Harness._p(r32), Harness._p(plain), Harness._p(shared), ctypes.c_uint64(len(r)))
        assert err == 0, "dh_alias: cudaError %d" % err
        p = r * n
        j = p >> 32
        frac = p & M32
        pr, al = prob_d[off + j], ali_d[off + j]
        want = torch.where((frac < pr) | (pr == M32), j, al)
        for name, got in (("alias_draw", plain), ("alias_draw_s", shared)):
            bad = torch.nonzero(got.to(torch.int64) != want)
            assert len(bad) == 0, "%s table %d word %#x: %d != %d" % (name, k, int(r[bad[0, 0]]), int(got[bad[0, 0]]), int(want[bad[0, 0]]))


@pytest.mark.gpu
def test_alias_all_words_realise_closed_form(device_lib):
    """All 2^32 words through alias_draw on the first-match table of guppy, counted on the device: the counts equal the
    closed form exactly, and agree with the float64 pmf within n 2^-32."""
    import torch

    t, desc = _alias_tables("guppy")
    alias, tab_off, tab_n = _alias_device(t)
    off, n = desc[0]
    counts = torch.zeros(n, dtype=torch.int64, device="cuda")
    err = device_lib.dh_alias_all_words(Harness._p(alias), Harness._p(tab_off), Harness._p(tab_n), ctypes.c_uint32(len(desc)),
                                        ctypes.c_uint32(0), Harness._p(counts))
    assert err == 0, "dh_alias_all_words: cudaError %d" % err
    got = counts.cpu().numpy()
    want = alias_exact_counts(t.alias_prob[off:off + n], t.alias_idx[off:off + n])
    np.testing.assert_array_equal(got, want)
    pmf = np.asarray(t.pmfs[0], dtype=np.float64)
    assert np.abs(got / 2.0 ** 32 - pmf / pmf.sum()).max() <= n * 2.0 ** -32


# ---------------------------------------------------------------------------------------------------------------------
# Box-Muller normal
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_box_muller_factors_and_realised_cdf(device_lib):
    """nf32_radius for all 2^24 values of r1 >> 8 and nf32_cos for all 2^24 values of r2 >> 8, each within 2 ulp of
    float64 (2^-24 absolute near 0); the CDF of z = radius * cos over all 2^48 pairs, in float64, within 1e-6 of Phi
    on t in [-6, 6]; |z| <= sqrt(48 ln 2); the cosines symmetric about 0."""
    import torch
    from scipy.special import ndtr

    radius = torch.empty(1 << 24, dtype=torch.float32, device="cuda")
    cosv = torch.empty(1 << 24, dtype=torch.float32, device="cuda")
    err = device_lib.dh_normal_factors(Harness._p(radius), Harness._p(cosv))
    assert err == 0, "dh_normal_factors: cudaError %d" % err
    v = np.arange(1 << 24, dtype=np.float64)
    r_ref = np.sqrt(-2.0 * np.log((v + 1.0) / 2.0 ** 24))
    c_ref = np.cos(2.0 * np.pi * v / 2.0 ** 24)
    for name, got, ref in (("radius", radius, r_ref), ("cos", cosv, c_ref)):
        g = got.cpu().numpy().astype(np.float64)
        tol = np.maximum(2.0 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64), 2.0 ** -24)
        e = np.abs(g - ref) / tol
        i = int(np.argmax(e))
        assert e[i] <= 1.0, "%s at v=%d: %.9g vs %.17g" % (name, i, g[i], ref[i])
    assert float(radius.max()) <= np.sqrt(48.0 * np.log(2.0)) * (1 + 2.0 ** -23) and float(cosv.abs().max()) <= 1.0
    cs = torch.sort(cosv.double()).values
    assert float((cs + cs.flip(0)).abs().max()) <= 2.0 ** -24                    # the multiset of cosines is symmetric
    rd = radius.double()
    grid = np.linspace(-6.0, 6.0, 121)
    worst = 0.0
    for x in grid:
        # P(z <= x) = 2^-24 sum over radius values of P(cos <= x / radius); radius 0 gives z = 0
        q = torch.where(rd > 0, x / rd, torch.full_like(rd, np.inf if x >= 0 else -np.inf))
        below = torch.searchsorted(cs, q, right=True).sum().item()
        cdf = below / 2.0 ** 48
        worst = max(worst, abs(cdf - float(ndtr(x))))
    assert worst <= 1e-6, "realised CDF of z differs from Phi by %.3g" % worst
