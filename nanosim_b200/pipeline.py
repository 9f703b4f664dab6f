"""Overlapped batch pipeline: the public way to run many batches.

``depth`` contexts (``ns_clone``: one copy of the reference and model in HBM, separate streams and batch buffers) are
driven by ``depth`` host threads (ctypes releases the GIL during library calls), so that while one batch is being copied
device->host into its pinned buffers the next batch's plan/emit kernels already run.  A context that finishes pulls the
next job at once (batches differ a lot in duration: unaligned batches are short and latency-bound), simulates it, and only
then waits for its pinned buffers to be released.  Results are handed to the consumer strictly in submission order,
which keeps output files identical to a sequential run.

This replaces the reference's ``for i in range(num_threads): mp.Process(...)`` fan-out
(/root/reference/src/simulator.py:1590-1622): same role (keep the machine busy), one GPU instead of N forks.
"""
import threading

import numpy as np

from . import _lib as L
from .engine import Batch


class _HostBuffers:
    """Pinned (page-locked) host buffers for one in-flight batch; grown on demand."""

    def __init__(self, fastq):
        self.fastq = fastq
        self.cap = {"seq": 0, "qual": 0, "reads": 0, "pieces": 0, "ops": 0, "gz": 0, "gz_err": 0}
        self.t = {}

    def _alloc(self, nbytes):
        try:
            import torch
            if torch.cuda.is_available():
                return torch.empty(int(nbytes), dtype=torch.uint8, pin_memory=True)
        except Exception:
            pass
        return np.empty(int(nbytes), dtype=np.uint8)

    def ensure(self, key, nbytes, hint=0):
        if nbytes > self.cap[key]:
            want = int(max(nbytes, hint) * 1.25) + 4096
            self.t[key] = self._alloc(want)
            self.cap[key] = want
        t = self.t[key]
        return t.numpy() if hasattr(t, "numpy") and not isinstance(t, np.ndarray) else t

    def ptr(self, key):
        t = self.t[key]
        return t.data_ptr() if hasattr(t, "data_ptr") else t.ctypes.data


class BatchPipeline:
    """compress: None, or names(batch, job) -> the batch's read names (records.NameTable).  With it the pipeline runs in
    compressed mode: the worker fetches the read and piece metadata (and the bases and ops when want_ops, for the error
    profile formatted on the host; never the qualities), builds the names, compresses the records on the device
    (ns_compress_records) and fetches the BGZF members into pinned memory; the consumer gets them as ``batch.gz`` and the
    names as ``batch.names``.  compress_profile (compressed mode, aligned batches): the error profile is formatted and
    compressed on the device as well (ns_compress_error_profile); its members arrive as ``batch.gz_err``.  bam
    (compressed mode): the records are unaligned BAM records (ns_compress_bam) instead of FASTA/FASTQ text.  mapped_bam (with
    bam): aligned batches are written as mapped BAM records (ns_compress_bam_mapped), unaligned ones stay unmapped;
    transcript_bam (with mapped_bam): against the transcripts (ns_compress_bam_transcript)."""

    def __init__(self, engine, depth=2, fetch=True, want_ops=False, want_pieces=True, compress=None, compress_profile=False,
                 bam=False, mapped_bam=False, transcript_bam=False):
        self.engines = [engine] + [engine.clone() for _ in range(max(1, depth) - 1)]
        self.depth = len(self.engines)
        self.fetch, self.want_ops, self.want_pieces, self.compress = fetch, want_ops, want_pieces, compress
        self.compress_profile, self.bam, self.mapped_bam, self.transcript_bam = compress_profile, bam, mapped_bam, transcript_bam
        self.bufs = [_HostBuffers(engine.fastq) for _ in self.engines]
        self.hint = {"seq": 0, "qual": 0, "reads": 0, "pieces": 0, "ops": 0, "gz": 0, "gz_err": 0}     # largest batch seen by any slot (pinned allocs are slow)

    def close(self):
        for e in self.engines[1:]:
            e.close()

    def _simulate(self, slot, job):
        kind, first, n = job
        return self.engines[slot].simulate(kind, first, n)

    def _pinned(self, slot, info):
        """take(key) -> the slot's pinned buffer ``key`` cut to the batch's bytes, grown for the largest batch any slot has seen."""
        nb = {"seq": int(info.seq_bytes), "qual": int(info.seq_bytes), "reads": int(info.n_reads) * L.READ_DTYPE.itemsize,
              "pieces": int(info.n_pieces) * L.PIECE_DTYPE.itemsize, "ops": int(info.n_ops) * 4}
        for k, v in nb.items():
            if v > self.hint[k]:
                self.hint[k] = v
        return lambda key: self.bufs[slot].ensure(key, nb[key], self.hint[key])[:nb[key]]

    def _fetch(self, slot, job, info):
        if self.compress is not None:
            return self._fetch_compressed(slot, job, info)
        kind, first, n = job
        eng, hb, take = self.engines[slot], self.bufs[slot], self._pinned(slot, info)
        fastq = eng.fastq
        seq = take("seq")
        qual = take("qual") if fastq else None
        reads = take("reads")
        pieces = take("pieces") if self.want_pieces else None
        ops = take("ops") if self.want_ops and info.n_ops else None
        eng.fetch_into(hb.ptr("seq"), hb.ptr("qual") if fastq else None, hb.ptr("reads"),
                       hb.ptr("pieces") if pieces is not None else None, hb.ptr("ops") if ops is not None else None)
        return Batch(info, seq, qual, reads.view(L.READ_DTYPE), pieces.view(L.PIECE_DTYPE) if pieces is not None else None,
                     ops.view(np.uint32) if ops is not None else np.zeros(0, dtype=np.uint32) if self.want_ops else None, kind, first)

    def _fetch_compressed(self, slot, job, info):
        kind, first, n = job
        eng, hb, take = self.engines[slot], self.bufs[slot], self._pinned(slot, info)
        reads = take("reads")
        pieces = take("pieces")
        seq = ops = None
        if self.want_ops:                  # the error-profile formatter reads bases back from the sequence
            seq = take("seq")
            if info.n_ops:
                ops = take("ops")
        eng.fetch_into(hb.ptr("seq") if seq is not None else None, None, hb.ptr("reads"), hb.ptr("pieces"),
                       hb.ptr("ops") if ops is not None else None)
        b = Batch(info, seq, None, reads.view(L.READ_DTYPE), pieces.view(L.PIECE_DTYPE),
                  ops.view(np.uint32) if ops is not None else np.zeros(0, dtype=np.uint32) if self.want_ops else None, kind, first)
        b.names = self.compress(b, job)
        if self.bam:
            mapped = self.mapped_bam and kind == L.NS_KIND_ALIGNED
            if not mapped:
                nz = eng.compress_bam(b.names)
            elif self.transcript_bam:
                nz = eng.compress_bam_transcript(b.names)
            else:
                nz = eng.compress_bam_mapped(b.names)
        else:
            nz = eng.compress_records(b.names)
        if nz > self.hint["gz"]:
            self.hint["gz"] = nz
        b.gz = eng.fetch_compressed(hb.ensure("gz", max(nz, 1), self.hint["gz"]))
        if self.compress_profile:
            ne = eng.compress_error_profile(b.names)
            if ne > self.hint["gz_err"]:
                self.hint["gz_err"] = ne
            b.gz_err = eng.fetch_compressed_error_profile(hb.ensure("gz_err", max(ne, 1), self.hint["gz_err"]))
        return b

    def warm(self, jobs):
        """Runs every job once on EVERY context (results discarded) so that device and pinned buffers reach their
        working size before anything is timed: growing a device buffer is a cudaFree + cudaMalloc, which synchronises
        the whole device and stalls the other contexts."""
        jobs = list(jobs)

        def one(slot):
            for job in jobs:
                info = self._simulate(slot, job)
                if self.fetch:
                    self._fetch(slot, job, info)

        threads = [threading.Thread(target=one, args=(s,), daemon=True) for s in range(self.depth)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()

    def run(self, jobs, consume=None, static_assign=False, after_simulate=None):
        """jobs: iterable of (kind, first_read_id, n_reads).  consume(info, batch, job) runs on the calling thread in
        submission order; the batch's buffers are reused as soon as consume returns.  Returns the list of infos.
        static_assign: job j always runs on context j % depth (needed when a context carries state from batch to batch,
        i.e. the metagenome species quotas) instead of on whichever context is free.
        after_simulate(engine, info, job) runs on the worker thread between the simulation and the fetch of a batch (the
        intron-retention pass patches reads there)."""
        jobs = list(jobs)
        n = len(jobs)
        results = [None] * n
        done = [threading.Event() for _ in range(n)]
        released = [threading.Event() for _ in range(self.depth)]     # the slot's pinned buffers may be overwritten
        for ev in released:
            ev.set()
        cursor = [0]
        lock = threading.Lock()
        errors = []

        def worker(slot):
            j = slot
            try:
                while True:
                    if static_assign:
                        if j >= n or errors:
                            return
                    else:
                        with lock:
                            j = cursor[0]
                            if j >= n or errors:
                                return
                            cursor[0] += 1
                    info = self._simulate(slot, jobs[j])
                    if after_simulate is not None:
                        after_simulate(self.engines[slot], info, jobs[j])
                        info = self.engines[slot].info
                    b = None
                    if self.fetch:
                        released[slot].wait()
                        released[slot].clear()
                        b = self._fetch(slot, jobs[j], info)
                    results[j] = (info, b, slot)
                    done[j].set()
                    if static_assign:
                        j += self.depth
            except BaseException as e:          # noqa: BLE001 -- re-raised on the calling thread
                errors.append(e)
                for ev in done:
                    ev.set()

        threads = [threading.Thread(target=worker, args=(s,), daemon=True) for s in range(min(self.depth, max(n, 1)))]
        for t in threads:
            t.start()
        infos = []
        try:
            for j in range(n):
                done[j].wait()
                if errors:
                    raise errors[0]
                info, b, slot = results[j]
                results[j] = None
                if consume is not None:
                    consume(info, b, jobs[j])
                infos.append(info)
                if self.fetch:
                    released[slot].set()
        finally:
            if len(infos) < n:
                errors.append(RuntimeError("pipeline aborted"))
                for ev in released:
                    ev.set()
            for t in threads:
                t.join()
        return infos
