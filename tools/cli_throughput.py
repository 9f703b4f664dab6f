"""Wall-clock of the CLI end to end (model load, simulation, formatting or compression, file writes) on the 5 Mb synthetic
reference, writing into /dev/shm when it exists.  Bases are counted from the reads files (text bytes / 2); a ``.gz`` file
(``--gzip``) is counted by its decompressed size, the sum of its BGZF members' ISIZE fields.  With --gzip the time of
every ns_compress_records call is reported too, and with --gzip_error_profile that of every ns_compress_error_profile call
(both calls end in a device synchronise) and the profile's compressed / plain ratio, next to zlib levels 1 and 6 on the
text of its first 1024 members (decompressed and compressed again on the CPU after the run).  With --bam every
ns_compress_bam call is timed, and the bases of a ``.bam`` file are the sum of its records' l_seq (read after the run)."""
import os, shutil, struct, sys, time, tempfile, zlib
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth
from nanosim_b200 import simulator
from nanosim_b200.engine import Engine


def text_bytes(path):
    """Bytes of the text a reads file holds: its size, or for BGZF (.gz, .bam) the sum of the members' ISIZE."""
    if not path.endswith((".gz", ".bam")):
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


def bam_bases(path):
    """Bases of a .bam reads file: the sum of its records' l_seq, inflating one BGZF member at a time."""
    total, buf, pos, header = 0, b"", 0, True
    with open(path, "rb") as f:
        while True:
            h = f.read(18)
            if len(h) < 18:
                return total
            size = struct.unpack("<H", h[16:18])[0] + 1
            buf = buf[pos:] + zlib.decompress(f.read(size - 18)[:-8], -15)
            pos = 0
            if header and len(buf) >= 8:
                l_text = struct.unpack_from("<i", buf, 4)[0]
                pos, header = 8 + l_text + 4, False          # magic, l_text, text, n_ref = 0
            while not header and pos + 24 <= len(buf):
                block = struct.unpack_from("<i", buf, pos)[0]
                if pos + 4 + block > len(buf):
                    break
                total += struct.unpack_from("<i", buf, pos + 20)[0]
                pos += 4 + block


def profile_sample(path, n_members=1024):
    """(compressed bytes, text) of the first n_members members after the header member of a .gz error profile."""
    data, pos, text, size = open(path, "rb").read(), 0, [], 0
    for k in range(n_members + 1):
        if pos >= len(data):
            break
        bsize = struct.unpack("<H", data[pos + 16:pos + 18])[0] + 1
        if k:
            text.append(zlib.decompress(data[pos:pos + bsize], 31))
            size += bsize
        pos += bsize
    return size, b"".join(text)


n = int(sys.argv[1]) if len(sys.argv) > 1 else 300000
extra = sys.argv[2:]
timings = {"ns_compress_records": [], "ns_compress_bam": [], "ns_compress_error_profile": []}


def timed(fn, key):
    def call(self, names):
        t = time.perf_counter()
        try:
            return fn(self, names)
        finally:
            timings[key].append(time.perf_counter() - t)
    return call


Engine.compress_records = timed(Engine.compress_records, "ns_compress_records")
Engine.compress_bam = timed(Engine.compress_bam, "ns_compress_bam")
Engine.compress_error_profile = timed(Engine.compress_error_profile, "ns_compress_error_profile")
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
    bases = sum(bam_bases(os.path.join(tmp, f)) if f.endswith(".bam") else text_bytes(os.path.join(tmp, f)) / 2 for f in reads)
    line = "CLI %d reads %s: %.1f s wall, ~%.2f Gbases, %.2f Gbases/s; files %s" % (
        n, extra, dt, bases / 1e9, bases / 1e9 / dt, {k: round(v / 1e9, 3) for k, v in sz.items()})
    if any(f.endswith((".gz", ".bam")) for f in reads):
        line += "; compressed / plain %.4f" % (sum(sz[f] for f in reads) / text)
    for key, c in timings.items():
        if c:
            c = sorted(c)
            line += "; %s %d calls, median %.1f ms, max %.1f ms, total %.2f s" % (key, len(c), 1e3 * c[len(c) // 2], 1e3 * c[-1], sum(c))
    err = os.path.join(tmp, "sim_aligned_error_profile.gz")
    if os.path.exists(err):
        line += "; error profile compressed / plain %.4f" % (sz["sim_aligned_error_profile.gz"] / text_bytes(err))
        size, sample = profile_sample(err)
        line += " (first %.0f MB of text: %.4f, zlib -1 %.4f, zlib -6 %.4f)" % (
            len(sample) / 1e6, size / len(sample), len(zlib.compress(sample, 1)) / len(sample), len(zlib.compress(sample, 6)) / len(sample))
    print(line)
finally:
    shutil.rmtree(tmp, ignore_errors=True)
