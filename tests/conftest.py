import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
ORACLE_DIR = os.path.join(ROOT, "oracle")
if ORACLE_DIR not in sys.path:
    sys.path.insert(0, ORACLE_DIR)

DATA = os.path.join(ROOT, "nanosim_b200", "data")
GOLDEN = os.path.join(ROOT, "tests", "golden")
MODEL_FILES = {"guppy": "guppy_fab49712_plusq.npz", "dorado": "dorado_kitv14_v3.2.1.npz",
               "even": "even_err3152364_v3.2.2.npz", "drna": "drna_bham1_guppy_plusq.npz"}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs at least two CUDA devices; not selected by -m gpu")


@pytest.fixture(scope="session")
def compiled_models():
    from nanosim_b200.model import CompiledModel

    return {k: CompiledModel.load(os.path.join(DATA, v)) for k, v in MODEL_FILES.items()}


def meta_fixture():
    """(OracleMetaReference, abundance numbers, {sample: {species: abundance}}) of tests/golden/meta."""
    import nanosim_oracle as no

    meta = os.path.join(GOLDEN, "meta")
    gl = os.path.join(meta, "genome_list_local.tsv")
    with open(os.path.join(meta, "genome_list.tsv")) as f, open(gl, "w") as o:
        for line in f:
            sp, path = line.rstrip("\n").split("\t")
            o.write("%s\t%s\n" % (sp, os.path.join(meta, os.path.basename(path))))
    ref = no.OracleMetaReference.from_genome_list(gl, os.path.join(meta, "dna_type.tsv"))
    numbers, multi = no.read_abundance(os.path.join(meta, "abundance.tsv"))
    return ref, numbers, multi


def oracle_model(cm, tmpdir, fastq=True, homopolymer=False, chimeric=False, perfect=False, mode="genome"):
    """Materialise a compiled model as reference-format text files and load it with the ORACLE's own
    parser; KDE samples come from the compiled model."""
    import nanosim_oracle as no

    prefix = os.path.join(str(tmpdir), "training")
    for name, text in cm.text.items():
        with open(prefix + "_" + name, "w") as f:
            f.write(text)
    m = no.OracleModel.load_text_tables(prefix, homopolymer=homopolymer, fastq=fastq, chimeric=chimeric, mode=mode)

    def kde(name):
        return no.OracleKDE(*cm.kde[name]) if name in cm.kde else None

    m.kde_ht = kde("ht_length")
    m.kde_ht_ratio = kde("ht_ratio")
    m.kde_unaligned = kde("unaligned_length")
    m.kde_gap = kde("gap_length")
    m.kde_aligned = kde("aligned_reads") if perfect else kde("aligned_region")
    m.kde_aligned_2d = kde("aligned_region_2d")
    return m
