"""Wall-clock of the CLI end to end (model load, simulation, formatting or compression, file writes) on the 5 Mb synthetic
reference, writing into /dev/shm when it exists.  Bases are counted from the reads files (text bytes / 2); a ``.gz`` file
(``--gzip``) is counted by its decompressed size, the sum of its BGZF members' ISIZE fields.  With --gzip the time of
every ns_compress_records call is reported too (the call ends in a device synchronise)."""
import os, shutil, struct, sys, time, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth
from nanosim_b200 import simulator
from nanosim_b200.engine import Engine


def text_bytes(path):
    """Bytes of the text a reads file holds: its size, or for BGZF the sum of the members' ISIZE."""
    if not path.endswith(".gz"):
        return os.path.getsize(path)
    total = 0
    with open(path, "rb") as f:
        while True:
            h = f.read(18)
            if len(h) < 18:
                return total
            size = struct.unpack("<H", h[16:18])[0] + 1
            f.seek(size - 18 - 4, 1)
            total += struct.unpack("<I", f.read(4))[0]


n = int(sys.argv[1]) if len(sys.argv) > 1 else 300000
extra = sys.argv[2:]
compress_s = []
_compress = Engine.compress_records


def timed_compress(self, names):
    t = time.perf_counter()
    try:
        return _compress(self, names)
    finally:
        compress_s.append(time.perf_counter() - t)


Engine.compress_records = timed_compress
tmp = tempfile.mkdtemp(prefix="cli_tp_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
try:
    ref = os.path.join(tmp, "ecoli5m.fa")
    synth.ecoli5m(ref)
    t0 = time.time()
    simulator.main(["genome", "-rg", ref, "-c", os.path.join(ROOT, "nanosim_b200", "data", "guppy_fab49712_plusq.npz"), "-n", str(n),
                    "-o", os.path.join(tmp, "sim"), "--fastq", "-t", "32", "--seed", "1"] + extra)
    dt = time.time() - t0
    reads = [f for f in os.listdir(tmp) if f.startswith("sim") and "_reads." in f]
    sz = {f: os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp) if f.startswith("sim")}
    text = sum(text_bytes(os.path.join(tmp, f)) for f in reads)
    bases = text / 2
    line = "CLI %d reads %s: %.1f s wall, ~%.2f Gbases, %.2f Gbases/s; files %s" % (
        n, extra, dt, bases / 1e9, bases / 1e9 / dt, {k: round(v / 1e9, 3) for k, v in sz.items()})
    if any(f.endswith(".gz") for f in reads):
        line += "; compressed / plain %.4f" % (sum(sz[f] for f in reads) / text)
    if compress_s:
        c = sorted(compress_s)
        line += "; ns_compress_records %d calls, median %.1f ms, max %.1f ms, total %.2f s" % (
            len(c), 1e3 * c[len(c) // 2], 1e3 * c[-1], sum(c))
    print(line)
finally:
    shutil.rmtree(tmp, ignore_errors=True)
