"""CPU tests of the host-side model compiler (nanosim_b200/model.py) against the oracle's own parsing/sampling."""
import os
import random

import numpy as np
import pytest

from conftest import DATA, oracle_model

import nanosim_oracle as no
from nanosim_b200 import model as M
from parity_checks import chi2_two_sample

CASES = ["guppy", "dorado"]


def _oracle_pmf(items):
    """Exact pmf of the oracle's interval sampler (all interval bounds are integers in shipped models)."""
    vmax = int(max(x[3] for x in items))
    pmf = np.zeros(vmax + 1)
    covered = 0.0
    for clo, chi, vlo, vhi in items:
        assert float(vlo).is_integer() and float(vhi).is_integer()
        n = int(vhi - vlo)
        covered += chi - clo
        if n == 0:
            pmf[int(vlo)] += chi - clo
        for s in range(int(vlo), int(vhi)):
            pmf[s] += (chi - clo) / n
    return pmf, covered


@pytest.mark.parametrize("tag", CASES)
def test_ecdf_pmfs_match_oracle_intervals(tag, compiled_models, tmp_path):
    cm = compiled_models[tag]
    om = oracle_model(cm, tmp_path, fastq=True)
    t = M.DeviceTables(cm, fastq=True)
    assert [tuple(b) for b in t.match_bins] == list(om.match_markov.keys())
    for b, pm in zip(om.match_markov.keys(), t.match_pmf):
        ref, covered = _oracle_pmf(om.match_markov[b])
        body = pm[:-1]
        assert len(body) == len(ref)
        np.testing.assert_allclose(body / body.sum(), ref / ref.sum(), atol=1e-13)
        # the miss slot is what the intervals leave uncovered
        assert abs(pm[-1] - max(0.0, 1.0 - covered)) < 1e-9
    fm_ref, _ = _oracle_pmf(om.first_match[list(om.first_match.keys())[0]])
    fm_ref[2] += fm_ref[0] + fm_ref[1]
    fm_ref[0] = fm_ref[1] = 0
    np.testing.assert_allclose(t.pmfs[M.T_FIRST][:len(fm_ref)], fm_ref / fm_ref.sum(), atol=1e-9)


@pytest.mark.parametrize("tag", CASES)
def test_alias_tables_realise_pmfs(tag, compiled_models):
    t = M.DeviceTables(compiled_models[tag], fastq=True)
    for i, pm in enumerate(t.pmfs):
        off, n = (int(x) for x in t.alias_desc[i])
        assert n == len(pm)
        got = M.alias_pmf(t.alias_prob[off:off + n], t.alias_idx[off:off + n])
        np.testing.assert_allclose(got, pm / pm.sum(), atol=2e-9)
        assert (t.alias_idx[off:off + n] < n).all()


@pytest.mark.parametrize("tag", CASES)
def test_error_length_pmfs_vs_oracle_sampling(tag, compiled_models, tmp_path):
    cm = compiled_models[tag]
    om = oracle_model(cm, tmp_path, fastq=True)
    t = M.DeviceTables(cm, fastq=True)
    n = 200000
    np.random.seed(5)
    random.seed(5)
    p = om.error_par["mis"]
    draws = {"mis": [no.pois_geom(p[0], p[2], p[3]) for _ in range(n)],
             "ins": [no.wei_geom(*om.error_par["ins"]) for _ in range(n)],
             "del": [no.wei_geom(*om.error_par["del"]) for _ in range(n)]}
    for tid, k in ((M.T_MIS, "mis"), (M.T_INS, "ins"), (M.T_DEL, "del")):
        pm = t.pmfs[tid]
        assert pm[0] == 0.0 and abs(pm.sum() - 1) < 1e-12
        emp = np.bincount(np.minimum(draws[k], len(pm) - 1), minlength=len(pm)).astype(float)
        stat, dof, pval = chi2_two_sample(emp, pm * 1e9)
        assert pval > 1e-4, (k, stat, dof, pval)


@pytest.mark.parametrize("tag", CASES)
def test_quality_pmf_vs_oracle_sampling(tag, compiled_models, tmp_path):
    cm = compiled_models[tag]
    om = oracle_model(cm, tmp_path, fastq=True)
    t = M.DeviceTables(cm, fastq=True)
    np.random.seed(9)
    for i, st in enumerate(M.QUAL_STATES):
        q = np.asarray(no.base_qualities(om.base_qual[st], 300000))
        assert q.min() >= 1 and q.max() <= 93
        emp = np.bincount(q, minlength=94).astype(float)
        stat, dof, pval = chi2_two_sample(emp, t.qual_pmf[i] * 1e10)
        assert pval > 1e-4, (st, stat, dof, pval)
        cdf = t.qual_cdf[i].astype(np.float64) / 2 ** 32
        np.testing.assert_allclose(np.diff(np.concatenate([[0], cdf])), t.qual_pmf[i], atol=1e-9)


@pytest.mark.parametrize("tag", CASES)
def test_transition_thresholds_and_counts(tag, compiled_models, tmp_path):
    cm = compiled_models[tag]
    om = oracle_model(cm, tmp_path, fastq=True)
    t = M.DeviceTables(cm, fastq=True)
    for i, st in enumerate(M.ERR_STATES):
        (a, b), (c, d), (e, f) = [iv for iv, _ in om.trans_error_pr[st]]
        assert abs(t.trans[i, 0] / 2 ** 32 - b) < 1e-9
        assert abs(t.trans[i, 1] / 2 ** 32 - d) < 1e-9
        assert abs(t.trans[i, 2] / 2 ** 32 - e) < 1e-9
    for n in (1000, 20000, 12345):
        assert t.split_counts(n) == om.split_counts(n)
    assert abs(t.strandness - om.strandness_rate) < 1e-7
    assert t.mean_ref_per_event > 1.0


def test_compiled_model_roundtrip(tmp_path, compiled_models):
    cm = compiled_models["guppy"]
    p = os.path.join(str(tmp_path), "m.npz")
    cm.save(p)
    cm2 = M.CompiledModel.load(p)
    assert cm2.text == cm.text
    for k in cm.kde:
        assert np.array_equal(cm.kde[k][0], cm2.kde[k][0]) and cm.kde[k][1] == cm2.kde[k][1]


def _new_obj(cls):
    return cls.__new__(cls)


class _EuclideanDistance:
    pickled_as = ("sklearn.neighbors._dist_metrics", "EuclideanDistance")

    def __reduce__(self):
        return _new_obj, (_EuclideanDistance,), (2.0, np.zeros(0), np.zeros((0, 0)))


class _KDTree:
    """The KDTree inside a scikit-learn 0.22/0.23 KernelDensity pickles as newObj(KDTree) + BinaryTree.__getstate__: (data,
    idx_array, node_data, node_bounds, leaf_size, n_levels, n_nodes, n_trims, n_leaves, n_splits, n_calls, dist_metric)."""
    pickled_as = ("sklearn.neighbors._kd_tree", "KDTree")

    def __init__(self, data):
        self.data = data

    def __reduce__(self):
        node = np.zeros(1, dtype=[("idx_start", "<i8"), ("idx_end", "<i8"), ("is_leaf", "<i8"), ("radius", "<f8")])
        bounds = np.stack([self.data.min(0), self.data.max(0)])[:, None, :]
        state = (self.data, np.arange(len(self.data), dtype=np.int64), node, bounds, 40, 1, 1, 0, 1, 0, 0,
                 _EuclideanDistance())
        return _new_obj, (_KDTree,), state


class _KernelDensity:
    pickled_as = ("sklearn.neighbors._kde", "KernelDensity")

    def __init__(self, data, bandwidth):
        self.__dict__.update(algorithm="auto", atol=0, bandwidth=bandwidth, breadth_first=True, kernel="gaussian",
                             leaf_size=40, metric="euclidean", metric_params=None, rtol=0, tree_=_KDTree(data))


_new_obj.pickled_as = ("sklearn.neighbors._kd_tree", "newObj")


def _dump_kde(path, data, bandwidth):
    """A ``<prefix>_<kde>.pkl`` as the reference's training writes it (joblib.dump of a KernelDensity), without sklearn."""
    import pickle
    from joblib.numpy_pickle import NumpyPickler

    class _Pickler(NumpyPickler):
        def save_global(self, obj, name=None):
            if not hasattr(obj, "pickled_as"):
                return super().save_global(obj, name)
            self.write(pickle.GLOBAL + ("%s\n%s\n" % obj.pickled_as).encode())
            self.memoize(obj)

    with open(path, "wb") as f:
        _Pickler(f, protocol=2).dump(_KernelDensity(data, bandwidth))


@pytest.mark.parametrize("tag,prefix", [("guppy", "training"), ("dorado", "hg002_nanosim_sub1M")])   # the archives' prefixes
def test_reference_model_directories_load_and_tabulate(tmp_path, tag, prefix):
    """`-c <model_dir>/<prefix>` on a model directory in the reference's format -- text tables + KernelDensity pickles --
    written from a shipped .npz: it loads back to exactly that model and tabulates into device tables."""
    from conftest import MODEL_FILES
    from nanosim_b200.model import CompiledModel, DeviceTables, load_model
    ours = CompiledModel.load(os.path.join(DATA, MODEL_FILES[tag]))
    prefix = os.path.join(str(tmp_path), prefix)
    for k, v in ours.text.items():
        with open(prefix + "_" + k, "w") as f:
            f.write(v)
    for k, (data, bw) in ours.kde.items():
        _dump_kde(prefix + "_" + k + ".pkl", data, bw)
    cm = load_model(prefix)
    t = DeviceTables(cm, fastq=False, chimeric="chimeric_info" in cm.text)
    assert len(t.alias_prob) > 1000 and len(cm.kde) >= 5
    assert cm.text == ours.text and sorted(cm.kde) == sorted(ours.kde)
    for k, (data, bw) in cm.kde.items():
        assert np.array_equal(ours.kde[k][0], data) and ours.kde[k][1] == bw, k
