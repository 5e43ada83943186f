"""PLINK 1 binary filesets (.bed / .bim / .fam) as a variants source.

The reference streams `Variant` records from the Google Genomics API (rdd/VariantsRDD.scala:187-236), which is retired;
cohorts of the size this path is built for live on disk as PLINK filesets or VCF.  A .bed file is already the packed
wire format of SURVEY.md 8f-1: variant-major, two bits per sample, four samples per byte (low bits first):

    0b00 homozygous A1   0b01 missing   0b10 heterozygous   0b11 homozygous A2        (A1, A2 = .bim columns 5, 6)

`hasVariation` (VariantsPca.scala:58, `genotype.foldLeft(false)(_ || _ > 0)`) becomes "carries the counted allele":
codes {00, 10} when A1 is counted (PLINK's default: A1 is the minor / alternate allele), {10, 11} when A2 is.  A missing
call is a no-call (-1, -1) and has no variation, exactly like the Scala rule.  Rows go to the GPU as they are on disk
(`NativePca.accumulateBed`, N/4 bytes per variant); `decode_rows` is the host-side statement of the same rule used by
`CallsRdd.collect()` and by the tests.
"""
from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Sequence, Tuple

import numpy as np

BED_MAGIC = bytes([0x6C, 0x1B, 0x01])          # 0x01 = variant-major
COUNT_A1, COUNT_A2 = 1, 2


def _prefix(path: str) -> str:
    p = str(path)
    for ext in (".bed", ".bim", ".fam"):
        if p.endswith(ext):
            return p[: -len(ext)]
    return p


def read_fam(path: str) -> List[Tuple[str, str]]:
    """[(callset id, callset name)] in file order.  id = "FID-IID" so that `callsetId.split("-").head`
    (VariantsPca.scala:235) yields the family id as the dataset column; name = IID."""
    out = []
    with open(_prefix(path) + ".fam", "r", encoding="utf-8") as fh:
        for line in fh:
            f = line.split()
            if len(f) >= 2:
                out.append((f"{f[0]}-{f[1]}", f[1]))
    if len({c[0] for c in out}) != len(out):
        raise ValueError(f"{path}: duplicate FID-IID in .fam")
    return out


def read_fam_ids(path: str) -> List[Tuple[str, str]]:
    """[(FID, IID)] (.fam columns 1 and 2) in file order."""
    with open(_prefix(path) + ".fam", "r", encoding="utf-8") as fh:
        return [(f[0], f[1]) for f in (line.split() for line in fh) if len(f) >= 2]


@dataclass(frozen=True)
class BimRecord:
    contig: str
    id: str
    position: int
    a1: str
    a2: str


def read_bim(path: str) -> List[BimRecord]:
    out = []
    with open(_prefix(path) + ".bim", "r", encoding="utf-8") as fh:
        for line in fh:
            f = line.split()
            if len(f) >= 6:
                out.append(BimRecord(f[0], f[1], int(f[3]), f[4], f[5]))
    return out


class BedFile:
    """Memory-mapped .bed: `rows(v0, v1)` is the (v1 - v0) x ceil(N / 4) uint8 block of variants [v0, v1)."""

    def __init__(self, path: str, n_samples: int | None = None, n_variants: int | None = None):
        self.prefix = _prefix(path)
        self.n_samples = n_samples if n_samples is not None else len(read_fam(self.prefix))
        self.stride = (self.n_samples + 3) // 4
        bed = Path(self.prefix + ".bed")
        size = bed.stat().st_size
        with open(bed, "rb") as fh:
            magic = fh.read(3)
        if magic[:2] != BED_MAGIC[:2]:
            raise ValueError(f"{bed}: not a PLINK .bed file")
        if magic[2:3] != BED_MAGIC[2:3]:
            raise ValueError(f"{bed}: sample-major .bed files are not supported (re-export with plink --make-bed)")
        if self.stride == 0 or (size - 3) % self.stride != 0:
            raise ValueError(f"{bed}: size {size} does not match {self.n_samples} samples")
        self.n_variants = (size - 3) // self.stride
        if n_variants is not None and n_variants != self.n_variants:
            raise ValueError(f"{bed}: {self.n_variants} variants on disk, {n_variants} in the .bim")
        self._map = np.memmap(bed, dtype=np.uint8, mode="r", offset=3, shape=(self.n_variants, self.stride)) \
            if self.n_variants else np.zeros((0, self.stride), np.uint8)

    def rows(self, v0: int, v1: int) -> np.ndarray:
        return np.ascontiguousarray(self._map[v0:v1])


def read_id_file(path: str) -> List[Tuple[Optional[str], str]]:
    """[(FID or None, IID)] of a sample ID file (--keep / --remove): whitespace-separated, blank lines ignored, a first line
    that starts with '#' is a header; a line gives FID IID as its first two tokens, or a bare IID as its only token.  This
    reads PLINK 2's `#FID IID` lists, such as .king.cutoff.in.id and .mindrem.id."""
    out: List[Tuple[Optional[str], str]] = []
    first = True
    with open(path, "r", encoding="utf-8") as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if first and tok[0].startswith("#"):
                first = False
                continue
            first = False
            out.append((tok[0], tok[1]) if len(tok) >= 2 else (None, tok[0]))
    return out


def sample_rows(fam_ids: Sequence[Tuple[str, str]], ids: Sequence[Tuple[Optional[str], str]], path: str = "ID file"):
    """(len(ids),) int64: the .fam sample each of read_id_file's entries names, -1 for none.  A bare IID matches the sample
    with that IID; it is refused (ValueError) when several families hold that IID."""
    pair = {fi: k for k, fi in enumerate(fam_ids)}
    by_iid: dict = {}
    for k, (_, iid) in enumerate(fam_ids):
        by_iid.setdefault(iid, []).append(k)
    out = np.full(len(ids), -1, np.int64)
    for j, (fid, iid) in enumerate(ids):
        if fid is None:
            ks = by_iid.get(iid, [])
            if len(ks) > 1:
                fams = ", ".join(fam_ids[k][0] for k in ks)
                raise ValueError(f"{path}: the bare IID {iid} is ambiguous: it occurs in families {fams}; give FID IID")
            k = ks[0] if ks else None
        else:
            k = pair.get((fid, iid))
        if k is not None:
            out[j] = k
    return out


def match_sample_ids(fam_ids: Sequence[Tuple[str, str]], ids: Sequence[Tuple[Optional[str], str]], path: str = "ID file"):
    """(listed (N,) bool over the .fam samples, IDs that match no sample) of read_id_file's entries (sample_rows' rule)."""
    rows = sample_rows(fam_ids, ids, path)
    listed = np.zeros(len(fam_ids), bool)
    listed[rows[rows >= 0]] = True
    return listed, int(np.count_nonzero(rows < 0))


MISSING_TOKENS = ("NA", "nan", "NaN", "-9")   # a missing value in a --pheno / --covar file


def read_value_file(path: str, stem: str):
    """A --pheno / --covar file -> (column names, [(FID or None, IID)], values (rows, columns) float64, NaN = missing).
    A first line `#FID IID ..`, `FID IID ..` or `#IID ..` is a header; without one every line is `FID IID v1 ..` and the
    columns are named stem1, stem2, ...  NA, nan and -9 are missing; any other value must be a finite number (ValueError
    naming the line otherwise), and every line must have the header's number of fields."""
    names, ids, values = None, [], []
    bare = False
    with open(path, "r", encoding="utf-8") as fh:
        for ln, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if names is None and not ids and tok[0] in ("#FID", "FID", "#IID"):
                bare = tok[0] == "#IID"
                names = tok[1:] if bare else tok[2:]
                continue
            first = 1 if bare else 2
            if names is None:
                names = [f"{stem}{c + 1}" for c in range(len(tok) - first)]
            if len(tok) != first + len(names):
                raise ValueError(f"{path}: line {ln} has {len(tok)} fields, {first + len(names)} expected")
            row = []
            for t in tok[first:]:
                if t in MISSING_TOKENS:
                    row.append(np.nan)
                    continue
                try:
                    x = float(t)
                except ValueError:
                    x = np.nan
                    t = None
                if t is None or not np.isfinite(x):
                    raise ValueError(f"{path}: line {ln}: {tok[first + len(row)]!r} is not a number (missing values are "
                                     f"{', '.join(MISSING_TOKENS)})")
                row.append(x)
            ids.append((None, tok[0]) if bare else (tok[0], tok[1]))
            values.append(row)
    if names is None:
        names = []
    if not names:
        raise ValueError(f"{path}: no value columns")
    return names, ids, np.asarray(values, np.float64).reshape(len(ids), len(names))


class SampleSubset:
    """The .bed rows of a fileset repacked to some of its samples (NativePca.subsetBedSamples), held in host memory, with
    the interface the driver reads from a BedFile; the prefix, and with it the .bim, stays the fileset's."""

    def __init__(self, bed: BedFile, keep_idx: np.ndarray, rows: np.ndarray):
        self.prefix = bed.prefix
        self.keep_idx = np.asarray(keep_idx, np.int64)
        self.n_samples = len(self.keep_idx)
        self.stride = (self.n_samples + 3) // 4
        self.n_variants = bed.n_variants
        if rows.shape != (self.n_variants, self.stride):
            raise ValueError(f"subset rows have shape {rows.shape}, not ({self.n_variants}, {self.stride})")
        self._map = rows

    def rows(self, v0: int, v1: int) -> np.ndarray:
        return np.ascontiguousarray(self._map[v0:v1])


@dataclass
class SampleSet:
    """The samples a --bed-path run analyses (--keep / --remove / --mind): the kept .fam entries in file order and the
    rows to read -- the fileset's own BedFile when every sample is kept, else a SampleSubset."""
    keep: np.ndarray                       # (N,) bool over the .fam samples
    callsets: List[Tuple[str, str]]        # read_fam entries of the kept samples
    fam_ids: List[Tuple[str, str]]         # read_fam_ids entries of the kept samples
    bed: object                            # BedFile | SampleSubset


def decode_rows(rows: np.ndarray, n_samples: int, counted: int = COUNT_A1) -> np.ndarray:
    """(nv, ceil(N/4)) uint8 -> (nv, N) bool `hasVariation` matrix (the rule in the module docstring)."""
    rows = np.asarray(rows, dtype=np.uint8)
    codes = np.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(rows.shape[0], -1)[:, :n_samples]
    if counted == COUNT_A1:
        return (codes == 0) | (codes == 2)
    if counted == COUNT_A2:
        return (codes == 2) | (codes == 3)
    raise ValueError("counted allele must be 1 (A1) or 2 (A2)")


def rows_to_calls(rows: np.ndarray, n_samples: int, counted: int = COUNT_A1):
    """The `RDD[Seq[Int]]` form (CSR offsets int64, idx int32) of a block of .bed rows; variants without any carrier are
    dropped, as VariantsPca.scala:166 does."""
    has = decode_rows(rows, n_samples, counted)
    has = has[has.any(axis=1)]
    counts = has.sum(axis=1)
    off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    idx = np.nonzero(has)[1].astype(np.int32)
    return off, idx


def window_starts(bim: Sequence[BimRecord], kb: float) -> np.ndarray:
    """(V,) int64 window_lo of LD pruning: the first variant i <= j on j's contig with pos_j - pos_i <= kb * 1000.
    Raises ValueError unless the contigs are contiguous runs and the positions do not decrease within a contig."""
    v = len(bim)
    lo = np.zeros(v, np.int64)
    pos = np.asarray([b.position for b in bim], np.int64)
    seen = set()
    r0 = 0
    while r0 < v:
        contig = bim[r0].contig
        if contig in seen:
            raise ValueError(f".bim is not sorted: contig {contig} comes back at variant {r0} ({bim[r0].id}, "
                             f"{contig}:{bim[r0].position}) after other contigs")
        seen.add(contig)
        r1 = r0 + 1
        while r1 < v and bim[r1].contig == contig:
            r1 += 1
        p = pos[r0:r1]
        down = np.flatnonzero(np.diff(p) < 0)
        if len(down):
            j = r0 + int(down[0]) + 1
            raise ValueError(f".bim is not sorted: variant {j} ({bim[j].id}, {contig}:{bim[j].position}) comes after "
                             f"{contig}:{bim[j - 1].position}")
        lo[r0:r1] = r0 + np.searchsorted(p, p - kb * 1000.0, side="left")
        r0 = r1
    return lo


def write_fileset(prefix: str, dosage_a1: np.ndarray, fam: Sequence[Tuple[str, str]] | None = None,
                  contig: str = "17", start: int = 41196311, *, contigs: Sequence[str] | None = None,
                  positions: Sequence[int] | None = None) -> None:
    """Write a fileset from an (N samples) x (V variants) array of A1 allele counts in {0, 1, 2} (-1 = missing);
    fam = [(FID, IID)] (default ("synth", "S000000"), ...).  Variant j sits on `contig` at start + j, or on contigs[j] at
    positions[j] when those are given.  Used by the tests and to export the synthetic cohort."""
    d = np.asarray(dosage_a1)
    n, v = d.shape
    code = np.full((v, n), 1, np.uint8)                     # missing
    dt = d.T
    code[dt == 2] = 0
    code[dt == 1] = 2
    code[dt == 0] = 3
    pad = (-n) % 4
    if pad:
        code = np.concatenate([code, np.zeros((v, pad), np.uint8)], axis=1)     # PLINK pads with 0 bits
    c4 = code.reshape(v, -1, 4)
    packed = (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)
    prefix = _prefix(prefix)
    with open(prefix + ".bed", "wb") as fh:
        fh.write(BED_MAGIC)
        fh.write(packed.tobytes())
    with open(prefix + ".bim", "w", encoding="utf-8") as fh:
        for j in range(v):
            c = contigs[j] if contigs is not None else contig
            pos = int(positions[j]) if positions is not None else start + j
            fh.write(f"{c}\trs{j + 1}\t0\t{pos}\tA\tG\n")
    with open(prefix + ".fam", "w", encoding="utf-8") as fh:
        for i in range(n):
            fid, iid = fam[i] if fam is not None else ("synth", f"S{i:06d}")
            fh.write(f"{fid} {iid} 0 0 0 -9\n")
