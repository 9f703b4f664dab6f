"""Reference loading: the product-side mirror of read_profile's FASTA half
(/root/reference/src/simulator.py:341-349 with readfq :709-740).

The sequence is kept exactly as in the file (case and IUPAC codes included) as one uint8 per base, all
chromosomes concatenated in file order; ``case_convert`` (:743-755) happens per read on the device, as in the
reference.  Chromosome keys follow :344-347: header up to the first space, ``[_\\s]`` runs replaced by ``-``,
truncated at the first ``.``.
"""
import re

import numpy as np


def normalise_name(header):
    raw = header.partition(" ")[0]
    return "-".join(re.split(r"[_\s]\s*", raw)).split(".")[0]


class PackedReference:
    def __init__(self, names, bases, offsets, raw_names=None):
        self.names = list(names)
        self.raw_names = list(raw_names) if raw_names is not None else list(names)   # header up to the first blank (pysam's view)
        self.bases = np.ascontiguousarray(bases, dtype=np.uint8)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        assert len(self.offsets) == len(self.names) + 1
        assert int(self.offsets[-1]) == len(self.bases)

    @property
    def lengths(self):
        return np.diff(self.offsets.astype(np.int64))

    @property
    def genome_len(self):
        return int(self.offsets[-1])

    @property
    def max_chrom(self):
        return int(self.lengths.max()) if len(self.names) else 0

    @staticmethod
    def from_records(records):
        """records: iterable of (header, uint8 array or bytes or str)."""
        names, parts, offs, raws = [], [], [0], []
        seen = {}
        for header, seq in records:
            if isinstance(seq, str):
                seq = seq.encode()
            arr = np.frombuffer(seq, dtype=np.uint8) if isinstance(seq, (bytes, bytearray)) else np.asarray(seq, dtype=np.uint8)
            key = normalise_name(header)
            if key in seen:             # seq_dict[key] = seqS: a repeated key overwrites the earlier record (:346)
                i = seen[key]
                parts[i] = arr
            else:
                seen[key] = len(names)
                names.append(key)
                raws.append(header.split()[0] if header.split() else header)
                parts.append(arr)
        for p in parts:
            offs.append(offs[-1] + len(p))
        bases = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
        return PackedReference(names, bases, np.asarray(offs, dtype=np.uint64), raws)

    @staticmethod
    def concat(a, b):
        """Records of `a` followed by the records of `b` (transcripts + the genome intron retention reads from)."""
        offs = np.concatenate([a.offsets, b.offsets[1:] + a.offsets[-1]]).astype(np.uint64)
        return PackedReference(a.names + b.names, np.concatenate([a.bases, b.bases]), offs, a.raw_names + b.raw_names)

    @staticmethod
    def from_fasta(path, n_threads=None):
        """FASTA (or FASTQ) file -> PackedReference.  The bytes are read by the library's multi-threaded mmap reader
        (ns_read_fasta); the pure-Python reader below is the fallback when the library is not built and for files with a
        repeated record key (a later record then replaces the earlier one, as seq_dict[key] = ... does, :346)."""
        try:
            ref = PackedReference._from_fasta_native(path, n_threads)
            if ref is not None:
                return ref
        except (OSError, RuntimeError):
            pass
        return PackedReference._from_fasta_python(path)

    @staticmethod
    def _from_fasta_native(path, n_threads=None):
        import ctypes as C
        import os

        from . import _lib
        lib = _lib.lib()
        nt = int(n_threads or min(32, os.cpu_count() or 1))
        n_rec, n_bases, hbytes = C.c_uint32(), C.c_uint64(), C.c_uint64()
        rc = lib.ns_read_fasta(os.fsencode(path), None, 0, None, None, 0, None, C.byref(n_rec), C.byref(n_bases), C.byref(hbytes), nt)
        if rc < 0:
            raise OSError("ns_read_fasta(%s) failed: %d" % (path, rc))
        bases = np.empty(n_bases.value, dtype=np.uint8)
        offs = np.zeros(n_rec.value + 1, dtype=np.uint64)
        hdr = np.zeros(max(hbytes.value, 1), dtype=np.uint8)
        hoff = np.zeros(max(n_rec.value, 1), dtype=np.uint64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = lib.ns_read_fasta(os.fsencode(path), vp(bases), len(bases), vp(offs), vp(hdr), len(hdr), vp(hoff), C.byref(n_rec),
                               C.byref(n_bases), C.byref(hbytes), nt)
        if rc < 0:
            raise OSError("ns_read_fasta(%s) failed: %d" % (path, rc))
        headers = [h.decode() for h in hdr.tobytes()[:hbytes.value].split(b"\0")[:n_rec.value]]
        names = [normalise_name(h) for h in headers]
        if len(set(names)) != len(names) or (n_rec.value and int(offs[0]) != 0):
            return None                       # repeated keys / bytes before the first record: the general path sorts it out
        raws = [h.split()[0] if h.split() else h for h in headers]
        return PackedReference(names, bases, offs, raws)

    @staticmethod
    def _from_fasta_python(path):
        with open(path, "rb") as f:
            blob = f.read()
        recs = []
        # records start at '>' at the beginning of a line
        starts = [0] if blob[:1] == b">" else []
        pos = blob.find(b"\n>")
        while pos != -1:
            starts.append(pos + 1)
            pos = blob.find(b"\n>", pos + 1)
        for i, s in enumerate(starts):
            e = starts[i + 1] if i + 1 < len(starts) else len(blob)
            nl = blob.find(b"\n", s, e)
            if nl == -1:
                nl = e
            header = blob[s + 1:nl].decode()
            body = blob[nl + 1:e].replace(b"\n", b"").replace(b"\r", b"")
            recs.append((header, body))
        return PackedReference.from_records(recs)


class MetaReference(PackedReference):
    """Metagenome reference (simulator.py:256-266, 284-339): species in genome-list order, the chromosomes of a species
    contiguous; chromosome names are ``{species}-{chrom}`` as in read names (:1747); per-chromosome circular/linear."""

    def __init__(self, names, bases, offsets, species, chrom_species, chrom_circular, chrom_keys):
        super().__init__(names, bases, offsets)
        self.species = list(species)
        self.chrom_species = np.ascontiguousarray(chrom_species, dtype=np.uint32)
        self.chrom_circular = np.ascontiguousarray(chrom_circular, dtype=np.uint8)
        self.chrom_keys = list(chrom_keys)

    @property
    def max_chrom_per_species(self):
        L = self.lengths
        return {sp: int(L[self.chrom_species == i].max()) for i, sp in enumerate(self.species)}

    @staticmethod
    def species_key(name):
        return "_".join(name.split())

    @staticmethod
    def from_genomes(genomes, dna_types=None):
        """genomes: ordered [(species, [(fasta header, sequence bytes/str/array), ...])]; dna_types: {species: {chrom: type}}."""
        names, parts, offs, sp_idx, circ, keys, species = [], [], [0], [], [], [], []
        for si, (sp, recs) in enumerate(genomes):
            sp = MetaReference.species_key(sp)
            species.append(sp)
            one = PackedReference.from_records(recs)
            for ci, key in enumerate(one.names):
                a, b = int(one.offsets[ci]), int(one.offsets[ci + 1])
                names.append(sp + "-" + key)
                keys.append(key)
                parts.append(one.bases[a:b])
                offs.append(offs[-1] + (b - a))
                sp_idx.append(si)
                ty = (dna_types or {}).get(sp, {}).get(key, "circular")      # local files default to circular (:323)
                circ.append(1 if ty == "circular" else 0)
        bases = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8)
        return MetaReference(names, bases, np.asarray(offs, dtype=np.uint64), species, sp_idx, circ, keys)

    @staticmethod
    def from_genome_list(genome_list, dna_type_list=None):
        genomes, raw_names = [], []
        with open(genome_list) as f:
            for line in f.readlines():
                if not line.strip():
                    continue
                fields = line.split("\t")
                path = fields[1].strip("\n")
                if path.startswith(("ftp", "http")):
                    raise ValueError("streaming reference genomes from RefSeq (simulator.py:295-315) is not supported")
                one = PackedReference.from_fasta(path)
                recs = [(k, one.bases[int(one.offsets[i]):int(one.offsets[i + 1])]) for i, k in enumerate(one.names)]
                genomes.append((fields[0], recs))
                raw_names += one.raw_names
        types = {}
        known = {MetaReference.species_key(g[0]) for g in genomes}
        if dna_type_list:
            with open(dna_type_list) as f:
                for line in f.readlines():
                    if not line.strip():
                        continue
                    fields = line.split("\t")
                    sp = MetaReference.species_key(fields[0])
                    if sp not in known:
                        raise KeyError("You didn't provide a reference genome for " + sp)
                    types.setdefault(sp, {})[normalise_name(fields[1])] = fields[2].strip("\n")
        m = MetaReference.from_genomes(genomes, types)
        m.raw_names = raw_names              # FASTA headers up to the first blank: the names a mapped BAM gives the records
        return m


def read_abundance(path, species):
    """Abundance table (simulator.py:360-380): header ``Size<TAB>n1<TAB>n2...``, one row per species.  Returns
    (number_list, [per-sample abundance vector in ``species`` order])."""
    with open(path) as f:
        header = f.readline()
        numbers = [int(x) for x in header.strip().split("\t")[1:]]
        table = {}
        for line in f.readlines():
            if not line.strip():
                continue
            fields = line.split("\t")
            if len(numbers) != len(fields) - 1:
                raise ValueError("Abundance file is incorrectly formatted. Check that each row has the same number of columns")
            sp = MetaReference.species_key(fields[0])
            if sp not in species:
                raise KeyError("You didn't provide a reference genome for " + sp)
            table[sp] = [float(x) for x in fields[1:]]
    # a species with a genome but no abundance row is simply not simulated (the reference leaves it out of dict_abun)
    samples = [[table[sp][i] if sp in table else 0.0 for sp in species] for i in range(len(numbers))]
    return numbers, samples


POLYA_SCALE = {"albacore": 2.409858743694814, "guppy": 4.168299657168961}      # simulator.py:1046-1049


def read_expression(path, ref):
    """Expression profile (simulator.py:385-401 + make_cdf :69-97): ``target_id est_counts tpm`` with a header; IDs are cut
    at the first '.'; transcripts with tpm > 0 that exist in the reference, with their TPM shares.
    Returns (expr_chrom uint32[n], weights float64[n])."""
    dict_exp = {}
    with open(path) as f:
        f.readline()
        for line in f:
            parts = line.split("\t")
            if len(parts) < 3:
                raise ValueError("Expression profile must contain 3 columns: ID, count, TPM ")
            tpm = float(parts[2])
            if tpm > 0:
                dict_exp[parts[0].split(".")[0]] = tpm
    if len(dict_exp) == 0:
        raise ValueError("Expression profile contains no TPM values > 0")
    index = {k: i for i, k in enumerate(ref.names)}
    chrom, w = [], []
    for tid, tpm in dict_exp.items():
        if tid in index:
            chrom.append(index[tid])
            w.append(tpm)
    if not chrom:
        raise ValueError("Please make sure transcript IDs in the expression profile match with those in reference "
                         "transcriptome (example: both Ensembl IDs)")
    w = np.asarray(w, dtype=np.float64)
    return np.asarray(chrom, dtype=np.uint32), w / w.sum()


def read_polya_list(path, ref):
    """--polya list (simulator.py:455-463): one transcript ID per line -> uint8 flag per reference record."""
    flags = np.zeros(len(ref.names), dtype=np.uint8)
    index = {k: i for i, k in enumerate(ref.names)}
    with open(path) as f:
        for line in f.readlines():
            i = index.get(line.strip().split(".")[0])
            if i is not None:
                flags[i] = 1
    return flags
