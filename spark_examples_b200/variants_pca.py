"""VariantsPcaDriver -- host-side mirror of the reference's driver class, same method names, argument
meaning and error behaviour (src/main/scala/com/google/cloud/genomics/spark/examples/VariantsPca.scala:36-288),
with the Spark map/reduceByKey similarity build (:182-191) and the MLlib eigen call (:224-227) replaced by the
CUDA path behind include/vpca.h.

    conf = PcaConf(["--synthetic", "2504,1000000"])
    driver = VariantsPcaDriver(conf)
    data = driver.getData
    filtered = [driver.filterDataset(d) for d in data]
    callsRdd = driver.getCallsRdd(filtered)
    simMatrix = driver.getSimilarityMatrix(callsRdd)
    result = driver.computePca(simMatrix)
    driver.emitResult(result)                     # VariantsPca.scala:38-50

Multi-GPU: launch one process per GPU (torchrun); partitions are dealt round-robin to the ranks and the partial
Grams are summed with ONE NCCL all-reduce -- the `reduceByKey(_ + _)` of :190.
"""
from __future__ import annotations

import dataclasses
import os
import struct
import sys
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import dist as vdist
from . import native
from .conf import PcaConf
from .jformat import jdouble
from .records import Call, CallData, Variant
from .parquet_calls import ParquetSlice
from .variants_common import BedSlice, CallsBatch, JoinedSlice, SyntheticSlice, VariantsCommon, VariantsDataset

MAX_LOADING_PC = 16   # components vpca_loadings_* / vpca_project_* handle (include/vpca.h)
SWAP_CODES = [3, 1, 2, 0]   # a z table indexed by the .bed code, re-indexed for the fileset with A1 and A2 swapped


# ------------------------------------------------------------------------------------------------------------------
# companion-object functions (VariantsPca.scala:54-78)
# ------------------------------------------------------------------------------------------------------------------
def extractCallInfo(variant: Variant, mapping: Dict[str, int]) -> List[CallData]:
    """VariantsPca.scala:56-60.  hasVariation = any allele index > 0 (a no-call, -1, is not variation); an unknown
    callset id raises KeyError, as `mapping(call.callsetId)` throws NoSuchElementException."""
    out = []
    for call in (variant.calls or ()):                      # variant.calls.getOrElse(Seq())
        has_variation = False
        for allele in call.genotype:                        # foldLeft(false)(_ || _ > 0)
            has_variation = has_variation or allele > 0
        out.append(CallData(has_variation, mapping[call.callsetId]))
    return out


def _fmix64(k: int) -> int:
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & 0xFFFFFFFFFFFFFFFF
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & 0xFFFFFFFFFFFFFFFF
    k ^= k >> 33
    return k


def _rotl64(x: int, r: int) -> int:
    return ((x << r) | (x >> (64 - r))) & 0xFFFFFFFFFFFFFFFF


def murmur3_128(data: bytes, seed: int = 0) -> str:
    """MurmurHash3_x64_128 -- what Guava's `Hashing.murmur3_128()` computes (un-vendored dependency, shaded at
    build.sbt:44); returns `HashCode.toString`: the 16 bytes (h1 then h2, little-endian) in hex."""
    c1, c2, M = 0x87C37B91114253D5, 0x4CF5AD432745937F, 0xFFFFFFFFFFFFFFFF
    h1 = h2 = seed & M
    n = len(data)
    nblocks = n // 16
    for i in range(nblocks):
        k1, k2 = struct.unpack_from("<QQ", data, i * 16)
        k1 = (k1 * c1) & M; k1 = _rotl64(k1, 31); k1 = (k1 * c2) & M; h1 ^= k1
        h1 = _rotl64(h1, 27); h1 = (h1 + h2) & M; h1 = (h1 * 5 + 0x52DCE729) & M
        k2 = (k2 * c2) & M; k2 = _rotl64(k2, 33); k2 = (k2 * c1) & M; h2 ^= k2
        h2 = _rotl64(h2, 31); h2 = (h2 + h1) & M; h2 = (h2 * 5 + 0x38495AB5) & M
    tail = data[nblocks * 16:]
    k1 = k2 = 0
    t = len(tail)
    if t > 8:
        k2 = int.from_bytes(tail[8:], "little")
        k2 = (k2 * c2) & M; k2 = _rotl64(k2, 33); k2 = (k2 * c1) & M; h2 ^= k2
    if t > 0:
        k1 = int.from_bytes(tail[:8], "little")
        k1 = (k1 * c1) & M; k1 = _rotl64(k1, 31); k1 = (k1 * c2) & M; h1 ^= k1
    h1 ^= n; h2 ^= n
    h1 = (h1 + h2) & M; h2 = (h2 + h1) & M
    h1 = _fmix64(h1); h2 = _fmix64(h2)
    h1 = (h1 + h2) & M; h2 = (h2 + h1) & M
    return (struct.pack("<QQ", h1, h2)).hex()


def variantKeyBytes(variant: Variant, debug: bool = False) -> bytes:
    """The bytes VariantsPca.scala:65-73 feeds the hasher: putString(contig), putLong(start), putLong(end),
    putString(referenceBases), putString(alternateBases.mkString("")) -- Guava writes longs little-endian."""
    alternate = "".join(variant.alternateBases) if variant.alternateBases is not None else ""
    reference = variant.referenceBases if variant.referenceBases is not None else ""
    if debug:
        print(f"{variant.contig}: ({variant.start}, {variant.end}) ref={reference} alt={alternate}")
    return (variant.contig.encode("utf-8") + struct.pack("<q", variant.start) + struct.pack("<q", variant.end) +
            reference.encode("utf-8") + alternate.encode("utf-8"))


def getVariantKey(variant: Variant, debug: bool = False) -> str:
    """VariantsPca.scala:62-78: murmur3_128 of contig, start, end, reference bases, joined alternate bases (host
    restatement; the product path hashes the same bytes on the GPU, vpca_hash_keys / vpca_join_rows)."""
    return murmur3_128(variantKeyBytes(variant, debug))


# ------------------------------------------------------------------------------------------------------------------
# RDD stand-ins
# ------------------------------------------------------------------------------------------------------------------
class CallsRdd:
    """`RDD[Seq[Int]]` (VariantsPca.scala:153): partitions of rows; a row lists the sample indices with variation."""

    def __init__(self, partitions: Sequence[object], n_samples: int):
        self.partitions = list(partitions)       # CallsBatch | SyntheticSlice | BedSlice
        self.n_samples = n_samples

    def collect(self) -> List[List[int]]:
        rows: List[List[int]] = []
        for p in self.partitions:
            if isinstance(p, SyntheticSlice):
                raise RuntimeError("synthetic partitions are generated on the device; use getSimilarityMatrix")
            if isinstance(p, BedSlice):
                from . import plink
                p = CallsBatch(*plink.rows_to_calls(p.rows(), self.n_samples, p.counted))
            if isinstance(p, ParquetSlice):
                p = p.load()
            if isinstance(p, JoinedSlice):
                p = joined_rows_on_host(p)
            for v in range(len(p.offsets) - 1):
                rows.append(p.idx[p.offsets[v]:p.offsets[v + 1]].tolist())
        return rows

    def count(self) -> int:
        return sum(p.n_rows if isinstance(p, BedSlice) else p.nv if isinstance(p, (SyntheticSlice, ParquetSlice))
                   else len(p.offsets) - 1 for p in self.partitions)


class SimilarityMatrix:
    """The `RDD[((Int, Int), Int)]` of VariantsPca.scala:182-191 (all N^2 keys present), resident on the GPU: it
    iterates / collects as ((row, col), count) records like the reference's RDD and additionally remembers the device
    handle, so `computePca` can run on the resident matrix without the N^2 records ever being materialised (the
    Scala twin is `GramRDD`, spark_examples_b200/jvm/GramRDD.scala)."""

    def __init__(self, nat: native.NativePca, n: int):
        self._nat, self.n = nat, n
        self._host: Optional[np.ndarray] = None

    def __iter__(self):
        S = self.toArray()
        for i in range(self.n):
            row = S[i]
            for j in range(self.n):
                yield ((i, j), int(row[j]))

    def toArray(self) -> np.ndarray:
        if self._host is None:
            self._host = self._nat.getGram()
        return self._host

    def collect(self) -> List[Tuple[Tuple[int, int], int]]:
        S = self.toArray()
        return [((i, j), int(S[i, j])) for i in range(self.n) for j in range(self.n)]


# ------------------------------------------------------------------------------------------------------------------
class VariantsPcaDriver:
    """VariantsPca.scala:81-286."""

    def __init__(self, conf: PcaConf, ctx=None, common: Optional[VariantsCommon] = None):
        self.conf = conf
        self.applicationName = type(self).__name__
        self._rank, self._world = vdist.rank_world()
        self.samples = None   # plink.SampleSet of --keep / --remove / --mind: every .fam read and fileset goes through it
        if common is None and sample_flags_given(conf):
            self.samples = self.selectSamples()
        self.common = common if common is not None else VariantsCommon(conf, ctx, samples=self.samples)
        self._nat: Optional[native.NativePca] = None
        self._gram_tensor = None
        self._torch_stream = None
        self._bim_cache: Dict[str, list] = {}
        self.pcaSamples: Optional[int] = None   # samples the last computePca solved for (fewer under --king-cutoff)
        self.grmUsed: Optional[int] = None      # M of the last --grm matrix

    # -- VariantsPca.scala:87 ---------------------------------------------------------------------------------------
    @property
    def getData(self) -> List[VariantsDataset]:
        return self.common.data

    # -- VariantsPca.scala:96-108 -----------------------------------------------------------------------------------
    def filterDataset(self, data: VariantsDataset) -> VariantsDataset:
        if not self.conf.minAlleleFrequency.isDefined:
            return data
        min_af = self.conf.minAlleleFrequency()
        print(f"Min allele frequency {np.float32(min_af)}.")                  # :99 (Float.toString)

        def keep(variant: Variant) -> bool:
            af = variant.info.get("AF")
            if af is None:
                return False                                  # getOrElse(false)
            return np.float32(float(af[0])) >= np.float32(min_af)   # .get(0).toFloat >= minAlleleFrequency

        def fn(part):
            if isinstance(part, (CallsBatch, SyntheticSlice, BedSlice, ParquetSlice)):
                raise ValueError("--min-allele-frequency needs Variant records (INFO field AF)")
            return [v for v in part if keep(v)]
        return data.map_partitions(fn)

    # -- VariantsPca.scala:115-148 ----------------------------------------------------------------------------------
    def joinDatasets(self, datasets: List[VariantsDataset]) -> List[List[CallData]]:
        """2-way join on the variant key (:115-128); calls of both sides concatenated (`related._1 ++ related._2`)."""
        mapping, debug = self.common.indexes, self.conf.debugDatasets()
        sides = []
        for ds in datasets[:2]:
            table: Dict[str, List[List[CallData]]] = {}
            for part in ds.partitions:
                for v in part:
                    table.setdefault(getVariantKey(v, debug), []).append(extractCallInfo(v, mapping))
            sides.append(table)
        out = []
        for key, left in sides[0].items():
            for l in left:                                      # inner join: cartesian product per key
                for r in sides[1].get(key, ()):
                    out.append(l + r)
        return out

    def mergeDatasets(self, datasets: List[VariantsDataset], variantSetCount: int) -> List[List[CallData]]:
        """N-way merge (:136-148): union, group by key, keep keys seen exactly `variantSetCount` times."""
        mapping = self.common.indexes
        groups: Dict[str, List[List[CallData]]] = {}
        for ds in datasets:
            for part in ds.partitions:
                for v in part:
                    groups.setdefault(getVariantKey(v), []).append(extractCallInfo(v, mapping))
        return [[c for calls in g for c in calls] for g in groups.values() if len(g) == variantSetCount]

    def _joined_slice(self, datasets: List[VariantsDataset], variantSetCount: int) -> JoinedSlice:
        """What joinDatasets / mergeDatasets shuffle, laid out for vpca_join_rows: per variant its key bytes (:65-73) and
        the callset indices with variation (:56-60, :164), datasets in order."""
        mapping, debug = self.common.indexes, self.conf.debugDatasets()
        join = variantSetCount == 2
        keys, lens, idx, n_left = [], [], [], 0
        for d, ds in enumerate(datasets[:2] if join else datasets):
            for part in ds.partitions:
                if isinstance(part, (CallsBatch, SyntheticSlice, BedSlice, ParquetSlice)):
                    raise ValueError("joining datasets needs Variant records (the key is made of contig / start / end / bases)")
                for v in part:
                    keys.append(variantKeyBytes(v, debug and join))
                    row = [c.callsetId for c in extractCallInfo(v, mapping) if c.hasVariation]
                    lens.append(len(row))
                    idx.extend(row)
            if d == 0:
                n_left = len(keys)
        off = np.zeros(len(keys) + 1, np.int64)
        np.cumsum(np.asarray(lens, np.int64), out=off[1:])
        return JoinedSlice(native.JOIN if join else native.MERGE, keys, off, np.asarray(idx, np.int32), n_left, variantSetCount)

    # -- VariantsPca.scala:153-168 ----------------------------------------------------------------------------------
    def getCallsRdd(self, data: List[VariantsDataset]) -> CallsRdd:
        n = len(self.common.indexes)
        # conf.variantSetId().size (:154); sources that are not API variant sets count the datasets they hold
        variantSetCount = len(self.conf.variantSetId()) if self.conf.variantSetId.isSupplied else len(data)
        mapping = self.common.indexes
        # loadings files key record rows by their variant key (:62-78); a projection keeps the rows without carriers,
        # which still contribute -mean * w
        want_keys = self.conf.saveLoadings.isDefined or self.conf.projectLoadings.isDefined
        if variantSetCount == 1:
            parts = []
            for part in data[0].partitions:
                if isinstance(part, (CallsBatch, SyntheticSlice, BedSlice, ParquetSlice)):
                    parts.append(part)                          # already RDD[Seq[Int]] rows (or their packed form)
                else:
                    keys = [variantKeyBytes(v) for v in part] if want_keys else None
                    parts.append(_rows_to_batch([extractCallInfo(v, mapping) for v in part], keys,
                                                keep_empty=self.conf.projectLoadings.isDefined))
            return CallsRdd(parts, n)
        # keying, join / merge and the concatenation of the calls run on the GPU and feed the encoder there (csrc/join.cu);
        # joinDatasets / mergeDatasets above stay as the record-level mirror of the reference's public methods
        return CallsRdd([self._joined_slice(data, variantSetCount)], n)

    # -- VariantsPca.scala:182-191 ----------------------------------------------------------------------------------
    def getSimilarityMatrix(self, callsets: CallsRdd) -> SimilarityMatrix:
        """S = sum over variants of x x^T on the GPU: every partition is one `mapPartitions` task (encode + wgmma
        Gram into a private staging Gram, committed on success); `reduceByKey(_ + _)` across ranks is one all-reduce."""
        if self.conf.grm():
            return self._getGrm(callsets)
        nat = self._native(callsets.n_samples)
        nat.reset()
        done = self._load_checkpoint(nat, callsets)
        for pid, part in enumerate(callsets.partitions):
            if vdist.partition_owner(pid, self._world) != self._rank or pid in done:
                continue
            if isinstance(part, SyntheticSlice):
                self._accumulate_synthetic(nat, part)
                continue
            if isinstance(part, ParquetSlice):
                part = part.load()                              # row group -> CSR rows, no per-record work
            try:
                if isinstance(part, JoinedSlice):
                    nat.joinRows(part.mode, part.keys, part.offsets, part.idx, part.n_left, part.variant_set_count)
                    nat.accumulateJoined(pid)                   # the joined rows never leave the device
                elif isinstance(part, BedSlice):
                    rows = part.rows()
                    if self.conf.makeKingTable.isDefined or self.conf.kingCutoff.isDefined:
                        nat.kinshipBed(rows)                    # the same rows, three genotype planes (DESIGN.md 7)
                    nat.accumulateBed(pid, rows, part.counted)
                else:
                    nat.accumulateCalls(pid, part.offsets, part.idx)
                nat.commit(pid)
            except Exception:
                nat.abort(pid)
                raise
            done.add(pid)
            self._save_checkpoint(nat, callsets, done, every=16)
        self._save_checkpoint(nat, callsets, done, every=1)
        if self._world > 1:
            # every count of the SUMMED matrix must stay a Java Int (VariantsPca.scala:185): bound it before the sum
            total = vdist.allreduce_count(nat.variantCount(), self._gram_tensor.device)
            if total * nat.max_multiplicity ** 2 > 2 ** 31 - 1:
                raise native.VpcaError(native.VPCA_ERR_OVERFLOW, f"{total} variants over all ranks could overflow an "
                                       "int32 similarity count")
            vdist.allreduce_gram(self._gram_tensor)            # VariantsPca.scala:190
        nat.finalizeGram()
        return SimilarityMatrix(nat, callsets.n_samples)

    def _getGrm(self, callsets: CallsRdd) -> SimilarityMatrix:
        """--grm: the variance-standardized relationship matrix of the .bed rows (DESIGN.md 13) instead of S, the KING
        counts riding on the same rows when asked for; writes P.rel.bin / P.rel.id with --make-rel before the solve."""
        nat = self._native(callsets.n_samples)
        nat.reset()
        V = 0
        for part in callsets.partitions:
            rows = part.rows()
            if self.conf.makeKingTable.isDefined:
                nat.kinshipBed(rows)
            nat.grmBed(rows)
            V += part.n_rows
        try:
            M = nat.grmFinalize()
        except native.VpcaError as e:
            if e.code != native.VPCA_ERR_STATE:
                raise
            raise ValueError(f"--grm: none of the {V} variants varies among its called samples (M = 0)") from None
        print(f"GRM: {M} of {V} variants used ({V - M} skipped: no variation among called samples).")
        self.grmUsed = M
        if self.conf.makeRel() and self._rank == 0:
            write_rel(self.conf.outputPath(), self._famIds(), nat.getGrm())
        return SimilarityMatrix(nat, callsets.n_samples)

    def getSimilarityMatrixStream(self, calls: CallsRdd) -> SimilarityMatrix:
        """VariantsPca.scala:262-279 yields the same matrix (its sparse-row quirk is not reproduced, SURVEY.md 2 row 3);
        on the GPU there is one implementation."""
        return self.getSimilarityMatrix(calls)

    # -- VariantsPca.scala:198-231 ----------------------------------------------------------------------------------
    def computePca(self, matrixEntries) -> List[Tuple[str, float, float]]:
        """`matrixEntries`: what getSimilarityMatrix returned (stays on the GPU), or -- the reference's signature,
        `RDD[((Int, Int), Int)]` (:198) -- any iterable of ((row, col), count) records, which are loaded into the GPU
        (absent keys count 0, like the rows `:216-221` never see)."""
        rowCount = len(self.common.indexes)
        numPc = self.conf.numPc()
        if numPc < 2:
            # the reference reads array(i + pca.numRows) (:230) and fails for numPc = 1
            raise IndexError("computePca reads the first two principal components; --num-pc must be >= 2")
        if isinstance(matrixEntries, SimilarityMatrix):
            nat = matrixEntries._nat
        else:
            S = np.zeros((rowCount, rowCount), np.int32)
            for (i, j), v in matrixEntries:
                S[i, j] = v                                                      # IndexError like Breeze at :216
            nat = self._native(rowCount)
            nat.setGram(S)
        if self.conf.grm():
            vecs, evals = nat.computePcaGrm(numPc)
            self.pcaSamples = rowCount
            if self.conf.outputPath.isDefined and self._rank == 0:
                write_eigen(self.conf.outputPath(), self._famIds(), vecs, evals)
        elif self.conf.kingCutoff.isDefined:
            vecs, evals, nonZeroRows = self._computePcaUnrelated(nat, rowCount, numPc)
        else:
            vecs, evals, nonZeroRows = nat.computePca(numPc)
            self.pcaSamples = rowCount
            print(f"Non zero rows in matrix: {nonZeroRows} / {rowCount}.")       # :208
        self.eigenvalues = evals
        self.components = vecs                                                   # all numPc columns (Python twin prints them)
        reverse = {i: cid for cid, i in self.common.indexes.items()}             # :228
        return [(reverse[i], float(vecs[i, 0]), float(vecs[i, 1])) for i in range(rowCount)]   # :229-230

    def _computePcaUnrelated(self, nat: native.NativePca, rowCount: int, numPc: int):
        """--king-cutoff X: the PCs of a maximal set of samples without a pair of KINSHIP > X, from the same Gram; every
        other sample is projected onto them from its Gram row (DESIGN.md 8).  The kinship counts rode on the Gram pass."""
        cutoff = self.conf.kingCutoff()
        ids, _, kin = nat.kinshipPairs(np.nextafter(cutoff, np.inf))              # exactly the pairs with KINSHIP > X
        keep = king_cutoff_keep(rowCount, ids, kin, cutoff)
        m = int(keep.sum())
        check_king_cutoff_kept(m, numPc)
        print(f"KING cutoff {cutoff!r}: {m} of {rowCount} samples kept, {rowCount - m} projected.")
        if self.conf.outputPath.isDefined and self._rank == 0:
            write_king_cutoff_ids(self.conf.outputPath(), self._famIds(), keep)
        vecs, evals, nonZeroRows = nat.computePcaSubset(keep, numPc)
        print(f"Non zero rows in matrix: {nonZeroRows} / {m}.")                  # :208, of the kept samples' matrix
        self.pcaSamples = m
        return vecs, evals, nonZeroRows

    # -- VariantsPca.scala:233-246 ----------------------------------------------------------------------------------
    def emitResult(self, result: Sequence[Tuple[str, float, float]], out=None):
        out = out or sys.stdout
        rows = []
        for callset_id, pc1, pc2 in result:
            dataset = callset_id.split("-")[0]                                   # :235
            rows.append((self.common.names[callset_id], pc1, pc2, dataset))
        if self._rank == 0:
            for name, pc1, pc2, dataset in sorted(rows, key=lambda t: t[0]):     # :238-239
                out.write(f"{name}\t{dataset}\t{jdouble(pc1)}\t{jdouble(pc2)}\n")
            if self.conf.outputPath.isDefined:                                   # :241-245 (saveAsTextFile layout)
                path = self.conf.outputPath() + "-pca.tsv"
                os.makedirs(path, exist_ok=True)
                with open(os.path.join(path, "part-00000"), "w", encoding="utf-8") as fh:
                    for name, pc1, pc2, dataset in rows:
                        fh.write(f"{name}\t{jdouble(pc1)}\t{jdouble(pc2)}\t{dataset}\n")
                open(os.path.join(path, "_SUCCESS"), "w").close()

    # -- variant loadings and projection onto saved principal coordinates (beyond :224-230; DESIGN.md 6) ------------
    def keyKind(self, callsets: CallsRdd) -> str:
        """How the rows of this cohort are identified in a loadings file: "variant" (murmur3_128 of the variant key,
        :62-78), "bim" (murmur3_128 of contig, position, A1, A2) or "row" (global row index)."""
        kinds = set()
        for p in callsets.partitions:
            if isinstance(p, JoinedSlice):
                raise ValueError("--save-loadings / --project-loadings read one dataset; joined multi-dataset input is "
                                 "not supported")
            kinds.add("bim" if isinstance(p, BedSlice) else
                      "variant" if isinstance(p, CallsBatch) and p.keys is not None else "row")
        if len(kinds) > 1:
            raise ValueError(f"partitions mix variant identities {sorted(kinds)}")
        return kinds.pop() if kinds else "row"

    @staticmethod
    def _counted_allele(callsets: CallsRdd) -> int:
        """1 / 2: .bed carriers of A1 / A2; 0: `hasVariation` of the calls (:58)."""
        for p in callsets.partitions:
            if isinstance(p, BedSlice):
                return int(p.counted)
        return 0

    def _partition_keys(self, part, row0: int) -> np.ndarray:
        """(nv, 2) uint64 identity of every row of a partition (see keyKind)."""
        if isinstance(part, BedSlice):
            return np.asarray([_hash_words(bimKeyBytes(b)) for b in self._partition_bim(part)], np.uint64).reshape(-1, 2)
        if isinstance(part, CallsBatch) and part.keys is not None:
            return np.asarray(part.keys, np.uint64).reshape(-1, 2)
        nv = _partition_len(part)
        keys = np.zeros((nv, 2), np.uint64)
        keys[:, 0] = np.arange(row0, row0 + nv, dtype=np.uint64)
        return keys

    def _partition_loadings(self, nat: native.NativePca, part, k: int, panel: int = 8192):
        if isinstance(part, SyntheticSlice):
            import torch
            dev = self._gram_tensor.device
            buf = torch.empty(nat.panelBytes(part.nv, panel), dtype=torch.uint8, device=dev)
            w = torch.empty((part.nv, k), dtype=torch.float64, device=dev)
            cnt = torch.empty(part.nv, dtype=torch.int32, device=dev)
            nat.synthPanelsDevice(part.seed, part.v0, part.nv, 0, buf.data_ptr(), panel)
            nat.loadingsPanels(k, buf.data_ptr(), part.nv, panel, w.data_ptr(), cnt.data_ptr())
            torch.cuda.current_stream().synchronize()
            return w.cpu().numpy(), cnt.cpu().numpy()
        if isinstance(part, BedSlice):
            return nat.loadingsBed(k, part.rows(), part.counted)
        off, idx = _partition_csr(part)
        return nat.loadingsCalls(k, off, idx)

    def saveLoadings(self, callsets: CallsRdd, path: Optional[str] = None):
        """After computePca: the loadings w = X^T U (numPc columns) and carrier counts of every variant of this run,
        streamed through the GPU a second time, written by rank 0 as one .npz (rows in partition order)."""
        path = path if path is not None else self.conf.saveLoadings()
        kind = self.keyKind(callsets)
        k = self.conf.numPc()
        starts = _partition_starts(callsets)
        mine = {}
        for pid, part in enumerate(callsets.partitions):
            if vdist.partition_owner(pid, self._world) != self._rank:
                continue
            w, cnt = self._partition_loadings(self._nat, part, k)
            mine[pid] = (self._partition_keys(part, starts[pid]), np.asarray(w, np.float64).reshape(-1, k),
                         np.asarray(cnt, np.int32))
        gathered = vdist.gather_to_rank0(mine)
        if self._rank != 0:
            return
        merged = {}
        for d in gathered:
            merged.update(d)
        order = sorted(merged)

        def cat(i, empty):
            return np.concatenate([merged[p][i] for p in order]) if order else empty
        with open(path, "wb") as fh:
            np.savez(fh, loadings=cat(1, np.zeros((0, k))), count=cat(2, np.zeros(0, np.int32)),
                     n_samples=np.int64(self.pcaSamples or len(self.common.indexes)), eigenvalues=np.asarray(self.eigenvalues[:k], np.float64),
                     counted_allele=np.int32(self._counted_allele(callsets)), keys=cat(0, np.zeros((0, 2), np.uint64)),
                     key_kind=np.str_(kind))

    def projectLoadings(self, callsets: CallsRdd, path: Optional[str] = None) -> List[Tuple[str, float, float]]:
        """Place this cohort in the PC space of a saved loadings file, without a Gram or an eigensolve: every row whose
        key is in the file goes through the GPU projection (rows without carriers too); file variants this cohort
        lacks contribute nothing (mean imputation).  Returns computePca's (callset id, pc1, pc2) rows."""
        path = path if path is not None else self.conf.projectLoadings()
        kind = self.keyKind(callsets)
        if loadings_matrix(path) == "grm":
            return self.projectGrmLoadings(callsets, path)
        with np.load(path, allow_pickle=False) as f:
            W, count, keys = f["loadings"], f["count"], f["keys"]
            n_ref, evals = int(f["n_samples"]), np.asarray(f["eigenvalues"], np.float64)
            file_kind, file_counted = str(f["key_kind"]), int(f["counted_allele"])
        if file_kind != kind:
            raise ValueError(f"{path} identifies variants by {file_kind!r} keys, this cohort's rows by {kind!r} keys")
        counted = self._counted_allele(callsets)
        if file_counted != counted:
            raise ValueError(f"{path} counts allele {file_counted}, this cohort counts allele {counted} (0: hasVariation)")
        k = W.shape[1] if W.ndim == 2 else 0
        if k < 2:
            raise ValueError(f"{path} holds {k} component(s); pc1 and pc2 need at least 2")
        mean = count.astype(np.float64) / n_ref
        index = {(int(a), int(b)): i for i, (a, b) in enumerate(keys)}
        rowCount = len(self.common.indexes)
        nat = self._native(rowCount)
        nat.reset()
        nat.projectBegin(k)
        starts = _partition_starts(callsets)
        for pid, part in enumerate(callsets.partitions):
            if vdist.partition_owner(pid, self._world) != self._rank:
                continue
            rows = np.asarray([index.get((int(a), int(b)), -1) for a, b in self._partition_keys(part, starts[pid])],
                              np.int64).reshape(-1)
            sel = rows >= 0
            if sel.any():
                self._partition_project(nat, part, sel, W[rows[sel]], mean[rows[sel]])
        if self._world > 1:
            raw = vdist.allreduce_f64(nat.projectGet(np.ones(k)), self._gram_tensor.device)
            P = raw / evals[None, :]
        else:
            P = nat.projectGet(evals)
        self.eigenvalues = evals
        self.components = P
        reverse = {i: cid for cid, i in self.common.indexes.items()}
        return [(reverse[i], float(P[i, 0]), float(P[i, 1])) for i in range(rowCount)]

    def _partition_project(self, nat: native.NativePca, part, sel: np.ndarray, w: np.ndarray, mean: np.ndarray,
                           panel: int = 8192):
        if isinstance(part, SyntheticSlice):
            # rows are born on the device: all of them go, unmatched rows with w = 0 and mean = 0
            import torch
            dev = self._gram_tensor.device
            W_full = np.zeros((part.nv, w.shape[1]), np.float64)
            m_full = np.zeros(part.nv, np.float64)
            W_full[sel], m_full[sel] = w, mean
            buf = torch.empty(nat.panelBytes(part.nv, panel), dtype=torch.uint8, device=dev)
            dw, dm = torch.from_numpy(W_full).to(dev), torch.from_numpy(m_full).to(dev)
            nat.synthPanelsDevice(part.seed, part.v0, part.nv, 0, buf.data_ptr(), panel)
            nat.projectPanels(buf.data_ptr(), part.nv, panel, dw.data_ptr(), dm.data_ptr())
            torch.cuda.current_stream().synchronize()       # the buffers must outlive the kernels that read them
        elif isinstance(part, BedSlice):
            nat.projectBed(part.rows()[sel], w, mean, part.counted)
        else:
            off, idx = _select_rows(*_partition_csr(part), sel)
            nat.projectCalls(off, idx, w, mean)

    # -- GRM loadings and projection onto the GRM's PCs (beyond the reference; DESIGN.md 14) ----------------------------
    def _partition_bim(self, part) -> list:
        """The .bim records of a BedSlice's rows (its kept rows only)."""
        from . import plink
        prefix = part.bed.prefix
        if prefix not in self._bim_cache:
            self._bim_cache[prefix] = plink.read_bim(prefix)
        bim = self._bim_cache[prefix][part.v0:part.v0 + part.nv]
        if part.keep is not None:
            bim = [b for b, k in zip(bim, part.keep.tolist()) if k]
        return bim

    def saveGrmLoadings(self, callsets: CallsRdd, path: Optional[str] = None):
        """After computePca of a --grm run: the GRM loadings w = Z^T U (numPc columns) and z tables of every variant of
        this run (after sample QC, variant QC and LD pruning), streamed through the GPU a second time, as one .npz."""
        path = path if path is not None else self.conf.saveGrmLoadings()
        kind = self.keyKind(callsets)
        k = self.conf.numPc()
        starts = _partition_starts(callsets)
        keys, ws, tabs = [], [], []
        for pid, part in enumerate(callsets.partitions):
            w, tab = self._nat.grmLoadingsBed(k, part.rows())
            keys.append(self._partition_keys(part, starts[pid]))
            ws.append(np.asarray(w, np.float64).reshape(-1, k))
            tabs.append(np.asarray(tab, np.float64).reshape(-1, 4))

        def cat(parts, empty):
            return np.concatenate(parts) if parts else empty
        with open(path, "wb") as fh:
            np.savez(fh, matrix=np.str_("grm"), loadings=cat(ws, np.zeros((0, k))), z_table=cat(tabs, np.zeros((0, 4))),
                     n_used=np.int64(self.grmUsed), eigenvalues=np.asarray(self.eigenvalues[:k], np.float64),
                     n_samples=np.int64(len(self.common.indexes)), keys=cat(keys, np.zeros((0, 2), np.uint64)),
                     key_kind=np.str_(kind))

    def projectGrmLoadings(self, callsets: CallsRdd, path: str) -> List[Tuple[str, float, float]]:
        """Place this cohort on the PCs of a saved GRM loadings file: p_c = sum_v tab[v][code] w[v][c] / (M lambda_c) over
        the file's variants found in this cohort by .bim key, or failing that with A1 and A2 swapped (then the table's
        HOM_A1 and HOM_A2 entries are exchanged, so the same allele is counted).  Strand-ambiguous pairs (A/T, C/G) are
        taken as given.  File variants this cohort lacks contribute nothing.  With --output-path P writes P.eigenvec."""
        with np.load(path, allow_pickle=False) as f:
            W, tab, keys = f["loadings"], f["z_table"], f["keys"]
            M, evals, file_kind = int(f["n_used"]), np.asarray(f["eigenvalues"], np.float64), str(f["key_kind"])
        kind = self.keyKind(callsets)
        if file_kind != kind:
            raise ValueError(f"{path} identifies variants by {file_kind!r} keys, this cohort's rows by {kind!r} keys")
        k = W.shape[1] if W.ndim == 2 else 0
        if k < 2:
            raise ValueError(f"{path} holds {k} component(s); pc1 and pc2 need at least 2")
        index = {(int(a), int(b)): i for i, (a, b) in enumerate(keys)}
        plan, found, swapped = [], 0, 0
        for part in callsets.partitions:
            bim = self._partition_bim(part)
            rows = np.asarray([index.get(_hash_words(bimKeyBytes(b)), -1) for b in bim], np.int64).reshape(-1)
            swap = np.zeros(len(rows), bool)
            for j in np.flatnonzero(rows < 0).tolist():   # a direct match wins; else the same variant with A1 / A2 swapped
                b = bim[j]
                i = index.get(_hash_words(bimKeyBytes(dataclasses.replace(b, a1=b.a2, a2=b.a1))), -1)
                if i >= 0:
                    rows[j], swap[j] = i, True
            sel = rows >= 0
            found += int(sel.sum())
            swapped += int(swap.sum())
            plan.append((part, sel, rows[sel], swap[sel]))
        print(f"GRM projection: {found} of {len(keys)} loadings variants found in this cohort "
              f"({swapped} with A1/A2 swapped).")
        if found == 0:
            raise ValueError(f"GRM projection: none of the {len(keys)} variants of {path} is in this cohort")
        rowCount = len(self.common.indexes)
        nat = self._native(rowCount)
        nat.reset()
        nat.projectBegin(k)
        for part, sel, rows, swap in plan:
            if not sel.any():
                continue
            t = tab[rows]
            t[swap] = t[swap][:, SWAP_CODES]
            nat.projectGrmBed(part.rows()[sel], t, W[rows])
        P = nat.projectGet(M * evals)
        self.eigenvalues = evals
        self.components = P
        if self.conf.outputPath.isDefined and self._rank == 0:
            write_eigenvec(self.conf.outputPath(), self._famIds(), P)
        reverse = {i: cid for cid, i in self.common.indexes.items()}
        return [(reverse[i], float(P[i, 0]), float(P[i, 1])) for i in range(rowCount)]

    # -- linear association tests with the PCs as covariates (beyond the reference; DESIGN.md 15) -------------------------
    def glmSamples(self, glm: "GlmInput") -> None:
        """Place the --pheno / --covar values on this run's samples (after sample QC), print how many IDs match none, and
        refuse too few regression samples or a phenotype of at most two values among them, before the Gram."""
        from . import plink
        # IDs are matched against the whole .fam, as --keep matches them, so only IDs absent from it count as unmatched;
        # an ID of a sample that sample QC removed matches and is dropped
        fam = plink.read_fam_ids(self.conf.bedPath())
        kept = self.samples.keep if self.samples is not None else np.ones(len(fam), bool)
        run_index = np.where(kept, np.cumsum(kept) - 1, -1)
        n = int(kept.sum())

        def place(ids, values, flag, path, out):
            rows = plink.sample_rows(fam, ids, f"{flag} {path}")
            found = rows >= 0
            at = np.full(len(rows), -1, np.int64)
            at[found] = run_index[rows[found]]
            out[at[at >= 0]] = values[at >= 0]
            return int(np.count_nonzero(~found))
        glm.y = np.full(n, np.nan)
        unmatched = {"--pheno": (glm.pheno_path, place(glm.pheno_ids, glm.pheno_values, "--pheno", glm.pheno_path,
                                                         glm.y))}
        glm.c = np.full((n, glm.covar_values.shape[1]), np.nan) if glm.covar_path else np.zeros((n, 0))
        if glm.covar_path:
            unmatched["--covar"] = (glm.covar_path, place(glm.covar_ids, glm.covar_values, "--covar", glm.covar_path,
                                                          glm.c))
        for flag, (path, k) in unmatched.items():
            if k:
                print(f"{flag} {path}: {k} IDs match no sample.")
        reg = np.isfinite(glm.y) & np.isfinite(glm.c).all(axis=1)
        if int(reg.sum()) < glm.q + 2:
            raise ValueError(f"--glm: {int(reg.sum())} of {n} samples have a phenotype and every covariate; {glm.q} "
                             f"covariates (the intercept included) need at least {glm.q + 2}")
        if glm.logistic:
            cases = int(np.count_nonzero(glm.y[reg] == 1.0))
            if cases == 0 or cases == int(reg.sum()):
                raise ValueError(f"--glm-logistic: phenotype {glm.name} has {cases} cases and {int(reg.sum()) - cases} "
                                 f"controls among the {int(reg.sum())} samples with a phenotype and every covariate; a "
                                 "logistic test needs both")
        else:
            check_glm_quantitative(glm.y[reg], glm.name)

    def _glmRun(self, callsets: CallsRdd, glm: "GlmInput", qc_keep, begin, bed, spec):
        """The driver loop of every association test: begin(nat, y, covariates) with the intercept, the run's PCs and the
        --covar columns as covariates, then bed(nat, rows, counted) on every variant that passes variant QC, in file
        order, on this run's rows.  spec: (dtype, shape of one variant's entry) of each output of bed.  Returns (the
        regression samples, the outputs concatenated over the partitions, the tested variants' .bim records, the
        counted allele, the covariates' description for the summary line)."""
        from . import plink
        pcs = np.asarray(self.components, np.float64)
        k = pcs.shape[1]
        nat = self._native(callsets.n_samples)
        used = begin(nat, glm.y, np.concatenate([pcs, glm.c], axis=1))
        chunks, tested = [], []
        counted = plink.COUNT_A1
        for part in callsets.partitions:
            sel = np.ones(part.nv, bool) if qc_keep is None else np.asarray(qc_keep[part.v0:part.v0 + part.nv], bool)
            rows = part.bed._map[part.v0:part.v0 + part.nv]        # read in place when every variant is tested
            chunks.append(bed(nat, rows if sel.all() else rows[sel], part.counted))
            tested.extend((part.v0 + np.flatnonzero(sel)).tolist())
            counted = part.counted
        outs = [np.concatenate([np.asarray(ch[i], t).reshape((-1,) + tail) for ch in chunks]) if chunks
                else np.zeros((0,) + tail, t) for i, (t, tail) in enumerate(spec)]
        bim = plink.read_bim(self.conf.bedPath())
        c = glm.c.shape[1]
        covs = f"{1 + k + c} covariates (intercept, {k} PCs" + (f", {c} from {glm.covar_path}" if glm.covar_path else "")
        return used, outs, [bim[j] for j in tested], counted, covs + ")"

    def glmLinear(self, callsets: CallsRdd, glm: "GlmInput", qc_keep: Optional[np.ndarray] = None):
        """After the PCs (or the projection): the linear test of every variant that passes variant QC, in file order, on
        this run's rows, with the intercept, the run's PCs and the --covar columns as covariates.  Writes
        P.<PHENO>.glm.linear and prints the `GLM linear:` line.  Returns (stats (V, 6), err (V,))."""
        used, (stats, errs), bim, counted, covs = self._glmRun(
            callsets, glm, qc_keep, lambda nat, y, c: nat.glmBegin(y, c), lambda nat, rows, a: nat.glmLinearBed(rows, a),
            ((np.float64, (6,)), (np.int32, ())))
        write_glm_linear(f"{self.conf.outputPath()}.{glm.name}.glm.linear", bim, counted, stats, errs)
        n = callsets.n_samples
        print(f"GLM linear: {glm.name} on {used} of {n} samples ({n - used} without a phenotype or covariate), "
              f"{covs}; {len(errs)} variants tested, {int(np.count_nonzero(errs))} with an "
              f"ERRCODE; lambda_GC = {lambda_gc(stats, errs)!r}.")
        return stats, errs

    def glmLogistic(self, callsets: CallsRdd, glm: "GlmInput", qc_keep: Optional[np.ndarray] = None):
        """glmLinear's logistic counterpart (DESIGN.md 16) for a case/control phenotype: writes P.<PHENO>.glm.logistic
        and prints the `GLM logistic:` line.  Returns (stats (V, 6), err (V,), passes (V,)).  With --glm-firth
        (DESIGN.md 17): fallback writes P.<PHENO>.glm.logistic.hybrid with the FIRTH? column and counts the Firth fits in
        the line; always writes P.<PHENO>.glm.firth and prints `GLM Firth:`."""
        spec = ((np.float64, (6,)), (np.int32, ()), (np.int32, ()))
        if glm.firth:
            bed = lambda nat, rows, a: nat.glmFirthBed(rows, a, glm.firth)   # noqa: E731
            spec += ((np.uint8, ()),)
        else:
            bed = lambda nat, rows, a: nat.glmLogisticBed(rows, a)   # noqa: E731
        used, outs, bim, counted, covs = self._glmRun(callsets, glm, qc_keep,
                                                      lambda nat, y, c: nat.glmLogisticBegin(y, c), bed, spec)
        stats, errs, passes = outs[:3]
        fitted = ""
        if glm.firth == "fallback":
            write_glm_logistic(f"{self.conf.outputPath()}.{glm.name}.glm.logistic.hybrid", bim, counted, stats, errs,
                               outs[3])
            fitted = f", {int(np.count_nonzero(outs[3]))} fitted by Firth regression"
        else:
            ext = "glm.firth" if glm.firth == "always" else "glm.logistic"
            write_glm_logistic(f"{self.conf.outputPath()}.{glm.name}.{ext}", bim, counted, stats, errs)
        n = callsets.n_samples
        reg = np.isfinite(glm.y) & np.isfinite(glm.c).all(axis=1)
        cases = int(np.count_nonzero(glm.y[reg] == 1.0))
        model = "Firth" if glm.firth == "always" else "logistic"
        print(f"GLM {model}: {glm.name} on {used} of {n} samples ({cases} cases, {used - cases} controls, {n - used} "
              f"without a phenotype or covariate), {covs}; {len(errs)} variants tested, "
              f"{int(np.count_nonzero(errs))} with an ERRCODE{fitted}; lambda_GC = {lambda_gc(stats, errs)!r}.")
        return stats, errs, passes

    # -- LD pruning of the variants (beyond the reference; DESIGN.md 9) -------------------------------------------------
    def ldPrune(self, callsets: CallsRdd, window_lo: np.ndarray, eligible: Optional[np.ndarray] = None) -> np.ndarray:
        """--ld-prune R2: keep-first LD pruning of the whole fileset in one library call; every BedSlice then stands for
        its kept rows only, so the Gram, the kinship counts and the loadings see the pruned variant set (what
        `plink --extract P.prune.in` would give).  eligible (the variant QC mask): prune only those variants, as PLINK
        does after its filters; the others are neither kept nor listed.  Returns the (V,) keep mask."""
        from . import plink
        r2, kb = self.conf.ldPrune(), self.conf.ldWindowKb()
        slices = [p for p in callsets.partitions if isinstance(p, BedSlice)]
        bed = slices[0].bed if slices else self._bedFile(callsets.n_samples)
        nat = self._native(callsets.n_samples)
        if eligible is None:
            keep, _, _ = nat.ldPruneBed(bed._map, window_lo, r2)
        else:
            keep, _, _ = nat.ldPruneBed(bed._map, window_lo, r2, eligible=eligible)
        of = len(keep) if eligible is None else int(np.count_nonzero(eligible))
        print(f"LD prune r2 > {r2!r} within {kb:g} kb: {int(keep.sum())} of {of} variants kept.")
        if self.conf.outputPath.isDefined and self._rank == 0:
            write_prune_lists(self.conf.outputPath(), plink.read_bim(self.conf.bedPath()), keep, eligible)
        for p in slices:
            p.keep = keep[p.v0:p.v0 + p.nv]
        return keep

    # -- variant QC (beyond the reference; DESIGN.md 10) --------------------------------------------------------------
    def variantQc(self, callsets: CallsRdd) -> np.ndarray:
        """--maf / --geno / --hwe: genotype counts and exact HWE p-values of the whole fileset in one library call; every
        BedSlice then stands for the variants that pass every filter given (what `plink --maf --geno --hwe --make-bed`
        would leave).  Writes P.afreq, P.vmiss and P.hardy with --output-path.  Returns the (V,) keep mask."""
        from . import plink
        slices = [p for p in callsets.partitions if isinstance(p, BedSlice)]
        bed = slices[0].bed if slices else self._bedFile(callsets.n_samples)
        nat = self._native(callsets.n_samples)
        counts, p = nat.variantQcBed(bed._map)
        limits = qc_limits(self.conf)
        keep, removed_by = variant_qc_keep(counts, p, limits["--maf"], limits["--geno"], limits["--hwe"])
        removed = ", ".join(f"{int(np.count_nonzero(removed_by == code))} by {flag} {limits[flag]!r}"
                            for code, flag in enumerate(QC_FILTERS, 1) if limits[flag] is not None)
        print(f"Variant QC: {int(keep.sum())} of {len(keep)} variants kept ({removed} removed).")
        if self.conf.outputPath.isDefined and self._rank == 0:
            write_qc_reports(self.conf.outputPath(), plink.read_bim(self.conf.bedPath()), counts, p)
        if not keep.any():
            raise ValueError(f"variant QC keeps none of the {len(keep)} variants ({removed}): relax --maf / --geno / --hwe")
        for s in slices:
            s.keep = keep[s.v0:s.v0 + s.nv]
        return keep

    # -- sample QC (beyond the reference; DESIGN.md 11) ----------------------------------------------------------------
    def selectSamples(self):
        """--keep / --remove / --mind: decide the samples of this --bed-path run before its context exists -> plink.SampleSet.
        The ID lists are matched on the host; --mind counts every sample's missing calls over all variants, and the rows
        are repacked to the kept samples, both on a short-lived 2-sample context (_sampleQcNative).  Every step below then
        sees a fileset of the kept samples only.  Prints the `Sample QC` line; writes P.smiss and P.mindrem.id with --mind
        and --output-path."""
        from . import plink
        conf, path = self.conf, self.conf.bedPath()
        callsets, fam_ids = plink.read_fam(path), plink.read_fam_ids(path)
        n = len(callsets)
        bed = plink.BedFile(path, n_samples=n)
        listed = {}
        for flag, opt in (("--keep", conf.keep), ("--remove", conf.remove)):
            if opt.isDefined:
                listed[flag], unmatched = plink.match_sample_ids(fam_ids, plink.read_id_file(opt()), f"{flag} {opt()}")
                if unmatched:
                    print(f"{flag} {opt()}: {unmatched} IDs match no sample.")
        keep, removed_by = sample_qc_keep(n, listed.get("--keep"), listed.get("--remove"))
        mind = conf.mind.get
        nat = None
        try:
            if mind is not None:
                nat = self._sampleQcNative()
                missing = np.asarray(nat.sampleMissingBed(bed._map, n), np.int64)
                left = keep.copy()
                keep, removed_by = sample_qc_keep(n, listed.get("--keep"), listed.get("--remove"), missing,
                                                  bed.n_variants, mind)
                if conf.outputPath.isDefined and self._rank == 0:
                    write_sample_qc_reports(conf.outputPath(), fam_ids, left, missing, bed.n_variants, removed_by == 3)
            m = int(keep.sum())
            given = {"--keep": "--keep" in listed, "--remove": "--remove" in listed, "--mind": mind is not None}
            removed = ", ".join(f"{int(np.count_nonzero(removed_by == code))} by {flag}" + (f" {mind!r}" if code == 3 else "")
                                for code, flag in enumerate(SAMPLE_FILTERS, 1) if given[flag])
            print(f"Sample QC: {m} of {n} samples kept ({removed} removed).")
            check_sample_kept(m, n, conf.numPc())
            check_king_flags(conf, m)                   # the kinship limit applies to the kept samples
            check_grm_flags(conf, m)
            if m == n:
                return plink.SampleSet(keep, callsets, fam_ids, bed)   # the fileset as it is
            kept = np.flatnonzero(keep)
            if nat is None:
                nat = self._sampleQcNative()
            rows = nat.subsetBedSamples(bed._map, n, kept)
        finally:
            if nat is not None:
                nat.close()
        return plink.SampleSet(keep, [callsets[k] for k in kept.tolist()], [fam_ids[k] for k in kept.tolist()],
                               plink.SampleSubset(bed, kept, rows))

    def _famIds(self) -> List[Tuple[str, str]]:
        """(FID, IID) of the samples of this run, in matrix order."""
        from . import plink
        return self.samples.fam_ids if self.samples is not None else plink.read_fam_ids(self.conf.bedPath())

    def _bedFile(self, n: int):
        """The fileset of this run's samples: its rows are what the Gram reads."""
        from . import plink
        return self.samples.bed if self.samples is not None else plink.BedFile(self.conf.bedPath(), n_samples=n)

    # -- KING-robust kinship of the sample pairs (beyond the reference; DESIGN.md 7) --------------------------------------
    def writeKingTable(self, path: Optional[str] = None, min_kinship: Optional[float] = None):
        """After getSimilarityMatrix of a --bed-path run with --make-king-table: rank 0 writes the pairs (filtered by
        --king-table-filter) in PLINK 2's .kin0 columns."""
        if self._rank != 0:
            return
        path = path if path is not None else self.conf.makeKingTable()
        if min_kinship is None:
            min_kinship = self.conf.kingTableFilter() if self.conf.kingTableFilter.isDefined else float("-inf")
        ids, counts, kin = self._nat.kinshipPairs(min_kinship)
        write_king_table(path, self._famIds(), ids, counts, kin)

    def reportIoStats(self):                                                     # :281
        self.common.reportIoStats()
        if self._nat is not None:
            st = self._nat.stats()
            print(f"GPU stats: variants={st['variants_accumulated']} gramLaunches={st['gram_launches']} "
                  f"kernelLaunches={st['kernel_launches']} h2dBytes={st['h2d_bytes']} lastGramMs={st['last_gram_ms']:.3f} "
                  f"lastEigMs={st['last_eig_ms']:.3f}")

    def stop(self):                                                              # :283-285
        if self._nat is not None:
            self._nat.close()
            self._nat = None

    # -- GPU plumbing --------------------------------------------------------------------------------------------
    def _device(self) -> int:
        return self.conf.gpuDevice() if self.conf.gpuDevice.isDefined else int(os.environ.get("LOCAL_RANK", "0"))

    def _sampleQcNative(self) -> native.NativePca:
        """The short-lived context of the sample QC calls, which read rows of any sample count: 2 samples (a few bytes of
        Gram), closed before the run's M-sample context and its M x M Gram exist."""
        return native.NativePca(2, device=self._device())

    def _native(self, n: int) -> native.NativePca:
        if self._nat is not None:
            return self._nat
        device = self._device()
        dtype = {"int8": native.DTYPE_I8, "i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16}[self.conf.gpuDtype()]
        stream = d_gram = 0
        try:
            import torch
            if torch.cuda.is_available():
                torch.cuda.set_device(device)
                self._torch_stream = torch.cuda.Stream(device=device)
                torch.cuda.set_stream(self._torch_stream)
                self._gram_tensor = torch.zeros((n, n), dtype=torch.int32, device=f"cuda:{device}")
                stream, d_gram = self._torch_stream.cuda_stream, self._gram_tensor.data_ptr()
        except ImportError:
            pass
        if self._world > 1 and d_gram == 0:
            raise RuntimeError("multi-rank runs need torch with CUDA for the NCCL all-reduce")
        self._nat = native.NativePca(n, device=device, dtype=dtype, num_pc=max(2, self.conf.numPc()), stream=stream,
                                     d_gram=d_gram)
        return self._nat

    # -- checkpoint / resume (SURVEY 8f-2): the natural checkpoint of this job is the int32 Gram (25 MB at N = 2504)
    #    plus the set of partitions already folded into it -- the counterpart of the reference's --input-path /
    #    --output-path persistence (GenomicsConf.scala:41,46).  One file per rank; partitions are committed atomically,
    #    so a file never holds a half-applied partition.
    def _checkpoint_file(self) -> Optional[str]:
        if not self.conf.checkpointPath.isDefined:
            return None
        return f"{self.conf.checkpointPath()}.rank{self._rank}of{self._world}.npz"

    def _load_checkpoint(self, nat: native.NativePca, callsets: CallsRdd) -> set:
        path = self._checkpoint_file()
        if path is None or not os.path.exists(path):
            return set()
        ck = np.load(path)
        if int(ck["n_samples"]) != callsets.n_samples or int(ck["n_partitions"]) != len(callsets.partitions):
            raise ValueError(f"checkpoint {path} belongs to a different cohort / partitioning")
        nat.loadPartialGram(ck["gram"], int(ck["variants"]))
        print(f"Resumed {len(ck['done'])} / {len(callsets.partitions)} partitions from {path}.")
        return set(int(p) for p in ck["done"])

    def _save_checkpoint(self, nat: native.NativePca, callsets: CallsRdd, done: set, every: int):
        path = self._checkpoint_file()
        if path is None or len(done) == 0 or len(done) % every:
            return
        tmp = path + ".tmp.npz"
        gram, variants = nat.partialGram(with_count=True)
        np.savez(tmp, gram=gram, variants=variants, done=np.array(sorted(done), np.int64), n_samples=callsets.n_samples,
                 n_partitions=len(callsets.partitions))
        os.replace(tmp, path)

    def _accumulate_synthetic(self, nat: native.NativePca, part: SyntheticSlice, panel: int = 8192):
        """Synthetic partitions are born on the device, directly in the panel layout the Gram kernel streams."""
        import torch
        buf = torch.empty(nat.panelBytes(part.nv, panel), dtype=torch.uint8, device=self._gram_tensor.device)
        nat.synthPanelsDevice(part.seed, part.v0, part.nv, 0, buf.data_ptr(), panel)
        nat.accumulatePanels(buf.data_ptr(), part.nv, panel)
        torch.cuda.current_stream().synchronize()      # `buf` must outlive the kernels that read it


KING_HEADER = "#FID1\tIID1\tFID2\tIID2\tNSNP\tHETHET\tIBS0\tKINSHIP\n"


def write_king_table(path: str, fam: Sequence[Tuple[str, str]], ids: np.ndarray, counts: np.ndarray,
                     kinship: np.ndarray, batch: int = 1 << 16) -> None:
    """Tab-separated KING table: one line per pair (ids[p] = (a, b), a < b; counts[p] = NSNP, HETHET, IBS0, HET1_HOM2,
    HET2_HOM1), FID / IID from .fam columns 1 and 2; KINSHIP as the shortest text that reads back as the same double."""
    with open(path, "w", encoding="utf-8") as fh:
        fh.write(KING_HEADER)
        for p0 in range(0, len(ids), batch):
            lines = []
            for (a, b), c, k in zip(ids[p0:p0 + batch].tolist(), counts[p0:p0 + batch].tolist(),
                                    kinship[p0:p0 + batch].tolist()):
                fa, fb = fam[a], fam[b]
                lines.append(f"{fa[0]}\t{fa[1]}\t{fb[0]}\t{fb[1]}\t{c[0]}\t{c[1]}\t{c[2]}\t{k!r}\n")
            fh.write("".join(lines))


def check_king_flags(conf: PcaConf, n_samples: Optional[int] = None) -> None:
    """Refuse --make-king-table / --king-table-filter / --king-cutoff runs the kinship path cannot serve, before any GPU
    work: without n_samples the flag combinations, with it the cohort size."""
    if conf.kingTableFilter.isDefined and not conf.makeKingTable.isDefined:
        raise ValueError("--king-table-filter needs --make-king-table")
    if conf.kingCutoff.isDefined and not np.isfinite(conf.kingCutoff()):
        raise ValueError(f"--king-cutoff must be a finite kinship, not {conf.kingCutoff()!r}")
    for flag, opt in (("--make-king-table", conf.makeKingTable), ("--king-cutoff", conf.kingCutoff)):
        if not opt.isDefined:
            continue
        if not conf.bedPath.isDefined:
            raise ValueError(f"{flag} needs genotype classes (het / hom): give a PLINK fileset with --bed-path")
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise ValueError(f"{flag} runs on one GPU; launch a single process (WORLD_SIZE=1)")
        if conf.checkpointPath.isDefined:
            raise ValueError(f"{flag} counts every partition in one pass; it cannot resume from --checkpoint-path")
        if conf.projectLoadings.isDefined:
            raise ValueError(f"--project-loadings builds no similarity matrix for {flag} to ride on")
        if n_samples is not None and n_samples > native.KINSHIP_MAX_SAMPLES:
            raise ValueError(f"{flag} is limited to {native.KINSHIP_MAX_SAMPLES} samples; the cohort has {n_samples}")


GRM_POINTERS = {
    "--king-cutoff": " (for the GRM PCs of an unrelated set, run --king-cutoff first and then --keep P.king.cutoff.in.id "
                     "--grm; its relatives go on those axes with --save-grm-loadings and --project-loadings)",
    "--save-loadings": " (the loadings of the GRM's PCs are written by --save-grm-loadings)",
    "--project-loadings": " (a GRM loadings file is projected without --grm: a projection builds no matrix)",
}


def loadings_matrix(path: str) -> str:
    """"grm" for a file of --save-grm-loadings, "carrier" for one of --save-loadings (which has no `matrix` field)."""
    with np.load(path, allow_pickle=False) as f:
        return str(f["matrix"]) if "matrix" in f.files else "carrier"


def check_projection_flags(conf: PcaConf) -> None:
    """Refuse a --project-loadings run of a GRM loadings file the GRM projection cannot serve, before any GPU work."""
    path = conf.projectLoadings.get
    if path is None or not os.path.exists(path) or loadings_matrix(path) != "grm":
        return                                          # (a missing file is reported where it is read)
    if not conf.bedPath.isDefined:
        raise ValueError(f"{conf.projectLoadings()} holds GRM loadings, which are projected from allele dosages: give a "
                         "PLINK fileset with --bed-path")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("projecting GRM loadings runs on one GPU; launch a single process (WORLD_SIZE=1)")


def check_grm_flags(conf: PcaConf, n_samples: Optional[int] = None) -> None:
    """Refuse --grm / --make-rel runs the GRM path cannot serve, before any GPU work: without n_samples the flag
    combinations, with it the cohort size."""
    if conf.makeRel() and not conf.grm():
        raise ValueError("--make-rel writes the matrix of --grm: give --grm")
    if conf.makeRel() and not conf.outputPath.isDefined:
        raise ValueError("--make-rel writes P.rel.bin and P.rel.id: give --output-path P")
    if conf.saveGrmLoadings.isDefined and not conf.grm():
        raise ValueError("--save-grm-loadings writes the loadings of --grm's PCs: give --grm")
    if not conf.grm():
        return
    if not conf.bedPath.isDefined:
        raise ValueError("--grm needs allele dosages: give a PLINK fileset with --bed-path")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("--grm runs on one GPU; launch a single process (WORLD_SIZE=1)")
    for flag, opt in (("--king-cutoff", conf.kingCutoff), ("--save-loadings", conf.saveLoadings),
                      ("--project-loadings", conf.projectLoadings), ("--checkpoint-path", conf.checkpointPath)):
        if opt.isDefined:
            raise ValueError(f"--grm cannot be combined with {flag}" + GRM_POINTERS.get(flag, ""))
    if conf.saveGrmLoadings.isDefined and conf.numPc() > MAX_LOADING_PC:
        raise ValueError(f"--save-grm-loadings stores at most {MAX_LOADING_PC} components; --num-pc {conf.numPc()} asks "
                         "for more")
    if n_samples is not None and n_samples > native.GRM_MAX_SAMPLES:
        raise ValueError(f"--grm is limited to {native.GRM_MAX_SAMPLES} samples; the cohort has {n_samples}")


def write_rel(prefix: str, fam: Sequence[Tuple[str, str]], G: np.ndarray) -> None:
    """--make-rel: prefix.rel.bin (N x N float64, little-endian, row-major: PLINK's `bin square`) and prefix.rel.id
    (`#FID<TAB>IID`, one line per sample in matrix order)."""
    np.ascontiguousarray(G, dtype="<f8").tofile(prefix + ".rel.bin")
    with open(prefix + ".rel.id", "w", encoding="utf-8") as fh:
        fh.write("#FID\tIID\n")
        fh.write("".join(f"{f}\t{i}\n" for f, i in fam))


def write_eigen(prefix: str, fam: Sequence[Tuple[str, str]], vecs: np.ndarray, evals: np.ndarray) -> None:
    """--grm with --output-path: prefix.eigenvec (write_eigenvec, the unit-norm eigenvectors) and prefix.eigenval (one
    eigenvalue per line), every number the shortest text that reads back as the same double."""
    write_eigenvec(prefix, fam, vecs)
    with open(prefix + ".eigenval", "w", encoding="utf-8") as fh:
        fh.write("".join(f"{x!r}\n" for x in np.asarray(evals, np.float64).tolist()))


def write_eigenvec(prefix: str, fam: Sequence[Tuple[str, str]], vecs: np.ndarray) -> None:
    """prefix.eigenvec: `#FID IID PC1 .. PCk`, tab-separated, one line per sample, every number the shortest text that
    reads back as the same double."""
    k = vecs.shape[1]
    with open(prefix + ".eigenvec", "w", encoding="utf-8") as fh:
        fh.write("#FID\tIID\t" + "\t".join(f"PC{c + 1}" for c in range(k)) + "\n")
        fh.write("".join(f"{f}\t{i}\t" + "\t".join(repr(x) for x in row) + "\n"
                         for (f, i), row in zip(fam, vecs.tolist())))


@dataclasses.dataclass
class GlmInput:
    """The --glm inputs read before any GPU work: the --pheno column and the --covar columns by file ID, and q (the
    intercept, the PCs and the covariates).  glmSamples sets y (N,) and c (N, columns) on the run's samples."""
    name: str
    pheno_path: str
    pheno_ids: list
    pheno_values: np.ndarray
    covar_path: Optional[str]
    covar_ids: list
    covar_values: np.ndarray
    q: int
    logistic: bool = False   # --glm-logistic: pheno_values hold 1 (case), 0 (control) and NaN (missing)
    firth: Optional[str] = None   # --glm-firth: "fallback" or "always"
    y: Optional[np.ndarray] = None
    c: Optional[np.ndarray] = None


LAMBDA_GC_DENOM = 0.45493642311957283   # the median of chi-square with 1 degree of freedom


def lambda_gc(stats: np.ndarray, errs: np.ndarray) -> float:
    """The genomic inflation factor: the median T_STAT^2 (Z_STAT^2 of a logistic test) over the variants without an
    ERRCODE / LAMBDA_GC_DENOM."""
    t = np.asarray(stats, np.float64)[np.asarray(errs) == 0, 4]
    return float(np.median(t * t) / LAMBDA_GC_DENOM) if len(t) else float("nan")


def check_glm_quantitative(values: np.ndarray, name: str) -> None:
    """Refuse a phenotype with at most two distinct values: a case/control trait, which linear regression does not fit."""
    distinct = np.unique(values[np.isfinite(values)])
    if len(distinct) <= 2:
        raise ValueError(f"--glm: phenotype {name} has {len(distinct)} distinct value(s); case/control traits need "
                         "logistic regression: add --glm-logistic")


def case_control_coding(values: np.ndarray, ids, name: str) -> np.ndarray:
    """PLINK's case/control coding -> 1 (case), 0 (control), NaN (missing): 2 is a case, 1 a control, and 0, -9, NA
    and nan are missing.  Any other value is refused with the sample's ID."""
    values = np.asarray(values, np.float64)
    out = np.full(len(values), np.nan)
    out[values == 2.0] = 1.0
    out[values == 1.0] = 0.0
    bad = np.flatnonzero(np.isfinite(values) & ~np.isin(values, (0.0, 1.0, 2.0, -9.0)))
    if len(bad):
        fid, iid = ids[bad[0]]
        who = iid if fid is None else f"{fid} {iid}"
        raise ValueError(f"--glm-logistic: phenotype {name} of sample {who} is {float(values[bad[0]])!r}; case/control "
                         "phenotypes are 1 (control), 2 (case), or 0, -9, NA or nan (missing)")
    return out


def check_glm_flags(conf: PcaConf) -> Optional[GlmInput]:
    """Refuse --glm / --pheno / --pheno-name / --covar runs the association path cannot serve, and read the phenotype
    and covariate files, before any GPU work.  Returns the inputs of a --glm run, else None."""
    for flag, opt in (("--pheno", conf.pheno), ("--pheno-name", conf.phenoName), ("--covar", conf.covar)):
        if opt.isDefined and not conf.glm():
            raise ValueError(f"{flag} is read by --glm: give --glm")
    if conf.glmLogistic() and not conf.glm():
        raise ValueError("--glm-logistic is a mode of --glm: give --glm")
    if conf.glmFirth.isDefined:
        if not (conf.glm() and conf.glmLogistic()):
            raise ValueError("--glm-firth is a mode of the logistic test: give --glm --glm-logistic")
        if conf.glmFirth() not in native.GLM_FIRTH_MODES:
            raise ValueError(f"--glm-firth takes fallback or always, not {conf.glmFirth()!r}")
    if not conf.glm():
        return None
    if not conf.pheno.isDefined:
        raise ValueError("--glm tests a phenotype: give --pheno FILE")
    if not conf.bedPath.isDefined:
        raise ValueError("--glm needs allele dosages: give a PLINK fileset with --bed-path")
    if not conf.outputPath.isDefined:
        raise ValueError("--glm writes P.<PHENO>.glm.linear: give --output-path P")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("--glm runs on one GPU; launch a single process (WORLD_SIZE=1)")
    if conf.checkpointPath.isDefined:
        raise ValueError("--glm tests the variants in one pass after the PCs; it cannot resume from --checkpoint-path")
    from . import plink
    names, ids, values = plink.read_value_file(conf.pheno(), "PHENO")
    name = conf.phenoName() if conf.phenoName.isDefined else names[0]
    if name not in names:
        raise ValueError(f"--pheno-name {name}: {conf.pheno()} has the columns {', '.join(names)}")
    y = values[:, names.index(name)]
    covar_ids, covar_values = [], np.zeros((0, 0))
    if conf.covar.isDefined:
        _, covar_ids, covar_values = plink.read_value_file(conf.covar(), "COVAR")
    if conf.projectLoadings.isDefined and os.path.exists(conf.projectLoadings()):
        with np.load(conf.projectLoadings(), allow_pickle=False) as f:
            k = int(f["loadings"].shape[1]) if "loadings" in f.files and f["loadings"].ndim == 2 else 0
        what = f"the {k} PCs of {conf.projectLoadings()}"
    else:
        k = conf.numPc()
        what = f"--num-pc {k}"
    q = 1 + k + covar_values.shape[1]
    if q > native.GLM_MAX_Q:
        raise ValueError(f"--glm fits at most {native.GLM_MAX_Q} covariates, the intercept included; the intercept, {what} "
                         f"and {covar_values.shape[1]} --covar columns make {q}")
    if conf.glmLogistic():
        return GlmInput(name, conf.pheno(), ids, case_control_coding(y, ids, name), conf.covar.get, covar_ids,
                        covar_values, q, logistic=True, firth=conf.glmFirth.get)
    check_glm_quantitative(y, name)
    return GlmInput(name, conf.pheno(), ids, y, conf.covar.get, covar_ids, covar_values, q)


def _glm_number(x: float) -> str:
    return "NA" if not np.isfinite(x) else repr(float(x))


def _glm_row_prefix(b, counted: int, st) -> str:
    """The first seven columns of a .glm.* row, through A1_FREQ and its tab."""
    return f"{b.contig}\t{b.position}\t{b.id}\t{b.a2}\t{b.a1}\t{b.a1 if counted == 1 else b.a2}\t{_glm_number(st[1])}\t"


def write_glm_linear(path: str, bim, counted: int, stats: np.ndarray, errs: np.ndarray) -> None:
    """P.<PHENO>.glm.linear, tab-separated, one line per tested variant in file order (PLINK 2's hide-covar columns): REF
    is A2 and ALT is A1 as in .afreq, A1 the counted allele, TEST ADD; numbers as the shortest text that reads back as the
    same double, NA where undefined."""
    with open(path, "w", encoding="utf-8") as fh:
        fh.write("#CHROM\tPOS\tID\tREF\tALT\tA1\tA1_FREQ\tTEST\tOBS_CT\tBETA\tSE\tT_STAT\tP\tERRCODE\n")
        fh.write("".join(
            f"{_glm_row_prefix(b, counted, st)}ADD\t{int(st[0])}\t{_glm_number(st[2])}\t{_glm_number(st[3])}\t{_glm_number(st[4])}\t"
            f"{_glm_number(st[5])}\t{native.GLM_ERRCODES[int(e)]}\n"
            for b, st, e in zip(bim, np.asarray(stats, np.float64).tolist(), np.asarray(errs).tolist())))


def write_glm_logistic(path: str, bim, counted: int, stats: np.ndarray, errs: np.ndarray,
                       firth: Optional[np.ndarray] = None) -> None:
    """P.<PHENO>.glm.logistic, as write_glm_linear with PLINK 2's logistic columns: OR = exp(BETA), LOG(OR)_SE = SE and
    Z_STAT in place of BETA, SE and T_STAT.  firth (the .hybrid file of --glm-firth fallback): a FIRTH? column after
    A1_FREQ, Y where the Firth fit produced the row."""
    fcol = "" if firth is None else "FIRTH?\t"
    flags = [""] * len(errs) if firth is None else ["Y\t" if f else "N\t" for f in np.asarray(firth).tolist()]
    with open(path, "w", encoding="utf-8") as fh:
        fh.write(f"#CHROM\tPOS\tID\tREF\tALT\tA1\tA1_FREQ\t{fcol}TEST\tOBS_CT\tOR\tLOG(OR)_SE\tZ_STAT\tP\tERRCODE\n")
        fh.write("".join(
            f"{_glm_row_prefix(b, counted, st)}{fl}ADD\t{int(st[0])}\t{_glm_number(np.exp(st[2]))}\t{_glm_number(st[3])}\t{_glm_number(st[4])}\t"
            f"{_glm_number(st[5])}\t{native.GLM_ERRCODES[int(e)]}\n"
            for b, st, e, fl in zip(bim, np.asarray(stats, np.float64).tolist(), np.asarray(errs).tolist(), flags)))


def check_ld_flags(conf: PcaConf, bim=None) -> Optional[np.ndarray]:
    """Refuse --ld-prune / --ld-window-kb runs the LD path cannot serve, before any GPU work: without `bim` the flag
    combinations, with the .bim records also their sort order and the window width.  Returns window_lo (with `bim`)."""
    if conf.ldWindowKb.isSupplied and not conf.ldPrune.isDefined:
        raise ValueError("--ld-window-kb needs --ld-prune")
    if not conf.ldPrune.isDefined:
        return None
    r2, kb = conf.ldPrune(), conf.ldWindowKb()
    if not (np.isfinite(r2) and 0.0 <= r2 < 1.0):
        raise ValueError(f"--ld-prune takes an r2 threshold in [0, 1), not {r2!r}")
    if not (np.isfinite(kb) and kb > 0):
        raise ValueError(f"--ld-window-kb must be a positive number of kb, not {kb!r}")
    if not conf.bedPath.isDefined:
        raise ValueError("--ld-prune needs allele counts and positions: give a PLINK fileset with --bed-path")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("--ld-prune runs on one GPU; launch a single process (WORLD_SIZE=1)")
    if conf.checkpointPath.isDefined:
        raise ValueError("--ld-prune decides the variant set before the Gram; it cannot resume from --checkpoint-path")
    if conf.projectLoadings.isDefined:
        raise ValueError("--project-loadings must use the reference's variants; drop --ld-prune")
    if bim is None:
        return None
    from . import plink
    try:
        lo = plink.window_starts(bim, kb)
    except ValueError as e:
        raise ValueError(f"--ld-prune needs a sorted .bim: {e}") from None
    reach = np.arange(len(lo), dtype=np.int64) - lo
    if len(reach) and reach.max() > native.LD_MAX_WINDOW:
        j = int(np.flatnonzero(reach > native.LD_MAX_WINDOW)[0])
        raise ValueError(f"--ld-window-kb {kb:g}: the window of variant {j} ({bim[j].id}, {bim[j].contig}:{bim[j].position}) "
                         f"holds {int(reach[j])} earlier variants; at most {native.LD_MAX_WINDOW} are supported")
    return lo


def write_prune_lists(prefix: str, bim, keep: np.ndarray, eligible: Optional[np.ndarray] = None) -> None:
    """PLINK's LD-pruning outputs: prefix.prune.in (the kept variants) and .prune.out (the pruned ones), the .bim variant
    IDs one per line in file order; with `eligible` (the variant QC mask) only eligible variants are listed."""
    keep = np.asarray(keep, bool)
    pruned = ~keep if eligible is None else np.asarray(eligible, bool) & ~keep
    for suffix, sel in ((".prune.in", keep), (".prune.out", pruned)):
        with open(prefix + suffix, "w", encoding="utf-8") as fh:
            fh.write("".join(f"{bim[j].id}\n" for j in np.flatnonzero(sel).tolist()))


QC_FILTERS = ("--geno", "--hwe", "--maf")   # PLINK's order: a removed variant is attributed to the first it fails
QC_RANGES = {"--maf": 0.5, "--geno": 1.0, "--hwe": 1.0}


def qc_limits(conf: PcaConf) -> Dict[str, Optional[float]]:
    """{flag: threshold or None} of the variant QC flags."""
    return {"--maf": conf.maf.get, "--geno": conf.geno.get, "--hwe": conf.hwe.get}


def check_qc_flags(conf: PcaConf) -> None:
    """Refuse --maf / --geno / --hwe runs the variant QC path cannot serve, before any GPU work."""
    given = [(flag, v) for flag, v in qc_limits(conf).items() if v is not None]
    if not given:
        return
    for flag, v in given:
        if not (np.isfinite(v) and 0.0 <= v <= QC_RANGES[flag]):
            raise ValueError(f"{flag} takes a value in [0, {QC_RANGES[flag]:g}], not {v!r}")
    flags = " / ".join(flag for flag, _ in given)
    if not conf.bedPath.isDefined:
        raise ValueError(f"{flags} counts genotypes: give a PLINK fileset with --bed-path")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError(f"{flags} runs on one GPU; launch a single process (WORLD_SIZE=1)")
    if conf.checkpointPath.isDefined:
        raise ValueError(f"{flags} decides the variant set before the Gram; it cannot resume from --checkpoint-path")
    if conf.projectLoadings.isDefined:
        raise ValueError(f"--project-loadings must use the reference's variants; drop {flags}")


def _allele_freqs(counts: np.ndarray):
    """(n called, A1 frequency f = (2 HOM_A1 + HET) / 2n, one rounded division; NaN when n = 0) of (V, 4) counts."""
    c = np.asarray(counts, np.int64).reshape(-1, 4)
    n = c[:, 0] + c[:, 1] + c[:, 2]
    with np.errstate(invalid="ignore", divide="ignore"):
        f = (2 * c[:, 0] + c[:, 1]).astype(np.float64) / (2 * n).astype(np.float64)
    return n, f


def variant_qc_keep(counts, p, maf: Optional[float], geno: Optional[float], hwe: Optional[float]):
    """(keep (V,) bool, removed_by (V,) int8) of (V, 4) counts (HOM_A1, HET, HOM_A2, MISSING) and HWE p-values (may be
    None without --hwe).  keep is the intersection of the filters given: --maf removes n = 0 or min(f, 1 - f) < maf,
    --geno removes MISSING / N > geno, --hwe removes p < hwe.  removed_by is 0 for a kept variant, else 1 + the index in
    QC_FILTERS of the first filter it fails."""
    c = np.asarray(counts, np.int64).reshape(-1, 4)
    n, f = _allele_freqs(c)
    fails = []
    if geno is not None:
        total = (n + c[:, 3]).astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            fails.append(c[:, 3].astype(np.float64) / total > geno)
    else:
        fails.append(np.zeros(len(c), bool))
    fails.append(np.asarray(p, np.float64) < hwe if hwe is not None else np.zeros(len(c), bool))
    if maf is not None:
        with np.errstate(invalid="ignore"):
            fails.append((n == 0) | (np.minimum(f, 1.0 - f) < maf))
    else:
        fails.append(np.zeros(len(c), bool))
    removed_by = np.zeros(len(c), np.int8)
    for code in (3, 2, 1):                          # the first filter failed wins
        removed_by[fails[code - 1]] = code
    return removed_by == 0, removed_by


def write_qc_reports(prefix: str, bim, counts, p) -> None:
    """PLINK 2's variant QC reports of every variant, tab-separated, in .bim order, doubles as the shortest text that
    reads back as the same double: prefix.afreq (A2 as REF, A1 as ALT, ALT_FREQS = the A1 frequency, OBS_CT = 2n),
    .vmiss (MISSING_CT, OBS_CT = N, F_MISS = MISSING_CT / N) and .hardy (O(HET_A1) = HET / n, E(HET_A1) = (2 f) (1 - f),
    P the exact HWE p-value)."""
    c = np.asarray(counts, np.int64).reshape(-1, 4)
    n, f = _allele_freqs(c)
    with np.errstate(invalid="ignore", divide="ignore"):
        total = n + c[:, 3]
        fmiss = c[:, 3].astype(np.float64) / total.astype(np.float64)
        o_het = c[:, 1].astype(np.float64) / n.astype(np.float64)
        e_het = (2.0 * f) * (1.0 - f)
    rows = list(zip(bim, c.tolist(), n.tolist(), f.tolist(), total.tolist(), fmiss.tolist(), o_het.tolist(),
                    e_het.tolist(), np.asarray(p, np.float64).tolist()))
    with open(prefix + ".afreq", "w", encoding="utf-8") as fh:
        fh.write("#CHROM\tID\tREF\tALT\tALT_FREQS\tOBS_CT\n")
        fh.write("".join(f"{b.contig}\t{b.id}\t{b.a2}\t{b.a1}\t{fr!r}\t{2 * nn}\n" for b, _, nn, fr, *_ in rows))
    with open(prefix + ".vmiss", "w", encoding="utf-8") as fh:
        fh.write("#CHROM\tID\tMISSING_CT\tOBS_CT\tF_MISS\n")
        fh.write("".join(f"{b.contig}\t{b.id}\t{cc[3]}\t{t}\t{fm!r}\n" for b, cc, _, _, t, fm, *_ in rows))
    with open(prefix + ".hardy", "w", encoding="utf-8") as fh:
        fh.write("#CHROM\tID\tA1\tAX\tHOM_A1_CT\tHET_A1_CT\tTWO_AX_CT\tO(HET_A1)\tE(HET_A1)\tP\n")
        fh.write("".join(f"{b.contig}\t{b.id}\t{b.a1}\t{b.a2}\t{cc[0]}\t{cc[1]}\t{cc[2]}\t{o!r}\t{e!r}\t{pp!r}\n"
                         for b, cc, _, _, _, _, o, e, pp in rows))


SAMPLE_FILTERS = ("--keep", "--remove", "--mind")   # a removed sample is attributed to the first that removes it


def sample_flags_given(conf: PcaConf) -> bool:
    return conf.keep.isDefined or conf.remove.isDefined or conf.mind.isDefined


def check_sample_flags(conf: PcaConf) -> None:
    """Refuse --keep / --remove / --mind runs the sample QC path cannot serve, before any GPU work.  An ID file that cannot
    be read is refused here; a bare IID that several families hold, when the .fam is matched (still before GPU work)."""
    given = [flag for flag, opt in zip(SAMPLE_FILTERS, (conf.keep, conf.remove, conf.mind)) if opt.isDefined]
    if not given:
        return
    if conf.mind.isDefined and not (np.isfinite(conf.mind()) and 0.0 <= conf.mind() <= 1.0):
        raise ValueError(f"--mind takes a value in [0, 1], not {conf.mind()!r}")
    flags = " / ".join(given)
    if not conf.bedPath.isDefined:
        raise ValueError(f"{flags} selects samples of a PLINK fileset: give --bed-path")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError(f"{flags} runs on one GPU; launch a single process (WORLD_SIZE=1)")
    if conf.checkpointPath.isDefined:
        raise ValueError(f"{flags} decides the samples before the Gram, and a checkpoint does not record them; drop "
                         "--checkpoint-path")
    from . import plink
    for flag, opt in (("--keep", conf.keep), ("--remove", conf.remove)):
        if opt.isDefined:
            try:
                plink.read_id_file(opt())
            except (OSError, UnicodeDecodeError) as e:
                raise ValueError(f"{flag} {opt()}: cannot read the ID file ({e})") from None


def sample_qc_keep(n: int, listed_keep=None, listed_remove=None, missing=None, n_variants: int = 0,
                   mind: Optional[float] = None):
    """(keep (N,) bool, removed_by (N,) int8) of the sample filters given: --keep keeps only listed_keep, --remove drops
    listed_remove, --mind drops F_MISS = MISSING_CT / V > mind (one rounded division; V = 0 removes nothing).  removed_by
    is 0 for a kept sample, else 1 + the index in SAMPLE_FILTERS of the first filter that removes it."""
    removed_by = np.zeros(n, np.int8)
    if listed_keep is not None:
        removed_by[~np.asarray(listed_keep, bool)] = 1
    if listed_remove is not None:
        removed_by[(removed_by == 0) & np.asarray(listed_remove, bool)] = 2
    if mind is not None:
        with np.errstate(invalid="ignore", divide="ignore"):
            fmiss = np.asarray(missing, np.int64).astype(np.float64) / np.float64(n_variants)
        removed_by[(removed_by == 0) & (fmiss > mind)] = 3
    return removed_by == 0, removed_by


def check_sample_kept(kept: int, n: int, num_pc: int) -> None:
    """Refuse a sample selection that leaves too few samples for the PCs asked for."""
    if kept < 2 or kept < num_pc:
        raise ValueError(f"sample QC keeps {kept} of {n} samples: at least max(2, --num-pc = {num_pc}) are needed")


def write_sample_qc_reports(prefix: str, fam: Sequence[Tuple[str, str]], left: np.ndarray, missing: np.ndarray,
                            n_variants: int, mind_removed: np.ndarray) -> None:
    """--mind's outputs: prefix.smiss (PLINK 2's columns, tab-separated: one line per sample left by --keep / --remove, in
    .fam order; OBS_CT = V, F_MISS = MISSING_CT / V as the shortest text that reads back as the same double) and
    prefix.mindrem.id (`#FID<TAB>IID`, the samples --mind removed; written even when empty)."""
    miss = np.asarray(missing, np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        fmiss = miss.astype(np.float64) / np.float64(n_variants)
    with open(prefix + ".smiss", "w", encoding="utf-8") as fh:
        fh.write("#FID\tIID\tMISSING_CT\tOBS_CT\tF_MISS\n")
        fh.write("".join(f"{fam[s][0]}\t{fam[s][1]}\t{int(miss[s])}\t{n_variants}\t{float(fmiss[s])!r}\n"
                         for s in np.flatnonzero(left).tolist()))
    with open(prefix + ".mindrem.id", "w", encoding="utf-8") as fh:
        fh.write("#FID\tIID\n")
        fh.write("".join(f"{fam[s][0]}\t{fam[s][1]}\n" for s in np.flatnonzero(mind_removed).tolist()))


def check_king_cutoff_kept(kept: int, num_pc: int) -> None:
    """Refuse a --king-cutoff selection that leaves too few samples for the PCs asked for."""
    if kept < 2 or kept < num_pc:
        raise ValueError(f"--king-cutoff keeps {kept} samples: at least max(2, --num-pc = {num_pc}) are needed")


def king_cutoff_keep(n: int, ids, kinship, cutoff: float) -> np.ndarray:
    """(n,) bool: a maximal set of samples without a pair of KINSHIP > cutoff (NaN is never related), chosen
    deterministically.  While related pairs remain, the sample with the most remaining related partners is removed (the
    larger index on a tie); then, in increasing index order, a removed sample returns when none of its relatives is in
    the set.  PLINK 2's --king-cutoff follows the same greedy idea; its tie-breaking is not reproduced."""
    ids = np.asarray(ids, np.int64).reshape(-1, 2)
    kin = np.asarray(kinship, np.float64).reshape(-1)
    partners: List[set] = [set() for _ in range(n)]
    for a, b in ids[kin > cutoff].tolist():
        if a != b:
            partners[a].add(b)
            partners[b].add(a)
    removed = np.zeros(n, bool)
    degree = np.array([len(p) for p in partners], np.int64)
    while n and degree.max() > 0:
        r = int(np.flatnonzero(degree == degree.max())[-1])
        removed[r] = True
        degree[r] = 0
        for j in partners[r]:
            if not removed[j]:
                degree[j] -= 1
    for r in np.flatnonzero(removed).tolist():
        if all(removed[j] for j in partners[r]):
            removed[r] = False
    return ~removed


def write_king_cutoff_ids(prefix: str, fam: Sequence[Tuple[str, str]], keep: np.ndarray) -> None:
    """PLINK 2's --king-cutoff outputs: prefix.king.cutoff.in.id (the kept samples) and .out.id (the removed ones),
    `#FID<TAB>IID` then one line per sample in fileset order."""
    keep = np.asarray(keep, bool)
    for suffix, sel in ((".king.cutoff.in.id", keep), (".king.cutoff.out.id", ~keep)):
        with open(prefix + suffix, "w", encoding="utf-8") as fh:
            fh.write("#FID\tIID\n")
            fh.write("".join(f"{fam[s][0]}\t{fam[s][1]}\n" for s in np.flatnonzero(sel).tolist()))


def joined_rows_on_host(p: JoinedSlice) -> CallsBatch:
    """The rows vpca_join_rows produces for `p`, computed with Python dicts (CallsRdd.collect and the tests' reference;
    same order: join by left row then right row, merge by first row of the group), empty rows dropped like :166."""
    rows = [p.idx[p.offsets[i]:p.offsets[i + 1]].tolist() for i in range(len(p.keys))]
    hashed = [murmur3_128(k) for k in p.keys]
    out: List[List[int]] = []
    if p.mode == native.JOIN:
        right: Dict[str, List[int]] = {}
        for j in range(p.n_left, len(rows)):
            right.setdefault(hashed[j], []).append(j)
        for i in range(p.n_left):
            for j in right.get(hashed[i], ()):
                out.append(rows[i] + rows[j])
    else:
        groups: Dict[str, List[int]] = {}
        for i, h in enumerate(hashed):
            groups.setdefault(h, []).append(i)
        for members in groups.values():
            if len(members) == p.variant_set_count:
                out.append([c for i in members for c in rows[i]])
    out = [r for r in out if len(r) > 0]
    off = np.zeros(len(out) + 1, np.int64)
    if out:
        off[1:] = np.cumsum([len(r) for r in out])
    return CallsBatch(off, np.asarray([c for r in out for c in r], np.int32))


def _rows_to_batch(rows: Iterable[Sequence[CallData]], keys: Optional[Sequence[bytes]] = None,
                   keep_empty: bool = False) -> CallsBatch:
    """VariantsPca.scala:164-167: keep calls with variation, drop empty variants, project to the callset index.
    keys: the variant key bytes of the rows (:65-73), hashed into CallsBatch.keys for the rows kept; keep_empty: keep
    the rows without carriers (a projection needs them)."""
    kept, kept_keys = [], []
    for v, calls in enumerate(rows):
        r = [c.callsetId for c in calls if c.hasVariation]
        if len(r) > 0 or keep_empty:
            kept.append(r)
            if keys is not None:
                kept_keys.append(_hash_words(keys[v]))
    off = np.zeros(len(kept) + 1, np.int64)
    if kept:
        off[1:] = np.cumsum([len(r) for r in kept])
        idx = np.concatenate([np.asarray(r, np.int32) for r in kept])
    else:
        idx = np.zeros(0, np.int32)
    if keys is None:
        return CallsBatch(off, idx)
    return CallsBatch(off, idx, np.asarray(kept_keys, np.uint64).reshape(-1, 2))


def _hash_words(key: bytes) -> Tuple[int, int]:
    """murmur3_128 of `key` as its two little-endian 64-bit halves (what vpca_hash_keys returns)."""
    h1, h2 = struct.unpack("<QQ", bytes.fromhex(murmur3_128(key)))
    return h1, h2


def bimKeyBytes(b) -> bytes:
    """Key bytes of a .bim record: contig, NUL, position (int64 little-endian), A1, NUL, A2."""
    return b.contig.encode("utf-8") + b"\0" + struct.pack("<q", b.position) + b.a1.encode("utf-8") + b"\0" + b.a2.encode("utf-8")


def _partition_len(part) -> int:
    if isinstance(part, BedSlice):
        return part.n_rows
    return len(part.offsets) - 1 if isinstance(part, CallsBatch) else int(part.nv)


def _partition_starts(callsets: CallsRdd) -> List[int]:
    """Global row index of the first row of every partition."""
    starts, r = [], 0
    for p in callsets.partitions:
        starts.append(r)
        r += _partition_len(p)
    return starts


def _partition_csr(part):
    """CSR rows of a calls partition; a Parquet row group keeps its rows without carriers (row keys stay aligned)."""
    if isinstance(part, ParquetSlice):
        return part.file.read_row_group(part.row_group)
    return part.offsets, part.idx


def _select_rows(off: np.ndarray, idx: np.ndarray, sel: np.ndarray):
    """The CSR rows where `sel` is true."""
    off = np.asarray(off, np.int64)
    counts = np.diff(off)
    row_of = np.repeat(np.arange(len(counts)), counts)
    new_off = np.zeros(int(sel.sum()) + 1, np.int64)
    np.cumsum(counts[sel], out=new_off[1:])
    return new_off, np.asarray(idx[off[0]:off[-1]], np.int32)[sel[row_of]]


def main(args: Optional[Sequence[str]] = None):
    """VariantsPcaDriver.main (VariantsPca.scala:38-50)."""
    conf = PcaConf(list(sys.argv[1:] if args is None else args))
    check_sample_flags(conf)
    check_king_flags(conf)
    check_grm_flags(conf)
    check_ld_flags(conf)
    check_qc_flags(conf)
    check_projection_flags(conf)
    glm = check_glm_flags(conf)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    driver = VariantsPcaDriver(conf)
    check_king_flags(conf, len(driver.common.indexes))
    check_grm_flags(conf, len(driver.common.indexes))
    if glm is not None:
        driver.glmSamples(glm)                          # after sample QC, before the Gram
    window_lo = None
    if conf.ldPrune.isDefined:
        from . import plink
        window_lo = check_ld_flags(conf, plink.read_bim(conf.bedPath()))
    data = driver.getData
    filtered = [driver.filterDataset(d) for d in data]
    callsRdd = driver.getCallsRdd(filtered)
    qc_keep = None
    if any(v is not None for v in qc_limits(conf).values()):
        qc_keep = driver.variantQc(callsRdd)            # the QC-passing set is the variant set of everything below
    if window_lo is not None:
        driver.ldPrune(callsRdd, window_lo, qc_keep)    # the pruned set is the variant set of everything below
    if conf.projectLoadings.isDefined:
        if conf.saveLoadings.isDefined:
            raise ValueError("--project-loadings computes no principal components to save; drop --save-loadings")
        result = driver.projectLoadings(callsRdd)
    else:
        if conf.saveLoadings.isDefined:
            if conf.numPc() > MAX_LOADING_PC:           # vpca_loadings_* take k <= 16: refuse before the Gram
                raise ValueError(f"--save-loadings stores at most {MAX_LOADING_PC} components; "
                                 f"--num-pc {conf.numPc()} asks for more")
            driver.keyKind(callsRdd)                    # reject unsupported input before the Gram
        simMatrix = driver.getSimilarityMatrix(callsRdd)
        result = driver.computePca(simMatrix)
        if conf.saveLoadings.isDefined:
            driver.saveLoadings(callsRdd)
        if conf.saveGrmLoadings.isDefined:
            driver.saveGrmLoadings(callsRdd)
    driver.emitResult(result)
    if glm is not None:
        if glm.logistic:
            driver.glmLogistic(callsRdd, glm, qc_keep)
        else:
            driver.glmLinear(callsRdd, glm, qc_keep)   # every QC-passing variant; the pruned set fed the PCs only
    if conf.makeKingTable.isDefined:
        driver.writeKingTable()
    driver.reportIoStats()
    driver.stop()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
