"""Multi-GPU product path (needs >= 2 GPUs: ``python -m pytest tests/test_multi_gpu.py``; on a box with fewer GPUs the one
test here is skipped for lack of hardware).

Two ranks under torchrun run the drop-in CLI: rank 0 alone reads the FASTA, the reference reaches rank 1's HBM through the
library's NCCL broadcast (ns_bcast_nccl), every rank simulates its shard of read ids and rank 0 concatenates the per-rank
files (/root/reference/src/simulator.py:1588-1639).  Reads are keyed by their global id, so the merged files must be
byte-identical to a single-process run."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

import parity_checks as pc
import synth

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_two_ranks_nccl_broadcast_equals_one_rank(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (this box has %d)" % torch.cuda.device_count())
    ref = os.path.join(str(tmp_path), "ecoli5m.fa")
    synth.ecoli5m(ref)
    model = os.path.join(pc.DATA, pc.MODELS["guppy"])
    args = ["genome", "-rg", ref, "-c", model, "-n", "4000", "--fastq", "--seed", "31", "--batch_reads", "700", "-t", "4"]
    one = os.path.join(str(tmp_path), "one")
    two = os.path.join(str(tmp_path), "two")
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-m", "nanosim_b200.simulator"] + args + ["-o", one], check=True, env=env, cwd=ROOT)
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                    "--master-port", "29741", "-m", "nanosim_b200.simulator"] + args + ["-o", two], check=True, env=env, cwd=ROOT)
    for suffix in ("_aligned_reads.fastq", "_unaligned_reads.fastq", "_aligned_error_profile"):
        a, b = open(one + suffix, "rb").read(), open(two + suffix, "rb").read()
        assert a == b and len(a) > 1000, suffix
    assert not os.path.exists(two + "_aligned_reads1.fastq")
