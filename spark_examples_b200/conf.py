"""Flag surface of the reference (Scallop option classes), kept name for name:
src/main/scala/com/google/cloud/genomics/spark/examples/GenomicsConf.scala:31-101.

Scallop derives `--kebab-case` flags from the camelCase vals (README.md:37-40); every option below is an
`Opt` that is called to read it (`conf.numPc()`) and has `.isDefined`, like a ScallopOption.  Options that
only exist here (GPU device/dtype, synthetic cohort) are additive.
"""
from __future__ import annotations

import argparse
import re
from typing import Any, List, Optional, Sequence


class GoogleGenomicsPublicData:
    """SearchVariantsExample.scala:27-31."""
    Platinum_Genomes = "3049512673186936334"
    Thousand_Genomes_Phase_1 = "10473108253681171589"
    Thousand_Genomes_Phase_3 = "4252737135923902652"


class Opt:
    """A parsed ScallopOption: call it for the value; `.isDefined` is true when supplied or defaulted."""

    def __init__(self, name: str, value: Any, supplied: bool):
        self.name, self._value, self.isSupplied = name, value, supplied

    @property
    def isDefined(self) -> bool:
        return self._value is not None

    def __call__(self):
        if self._value is None:
            raise KeyError(f"option --{self.name} is not defined")     # Scallop throws on apply() of an empty option
        return self._value

    @property
    def get(self):
        return self._value

    def __repr__(self):
        return f"Opt({self.name}={self._value!r})"


def _kebab(name: str) -> str:
    return re.sub(r"(?<!^)(?=[A-Z])", "-", name).lower()


class GenomicsConf:
    """GenomicsConf.scala:31-70."""
    DEFAULT_NUMBER_OF_BASES_PER_SHARD = 1000000
    PLATINUM_GENOMES_BRCA1_REFERENCES = "chr17:41196311:41277499"

    def _options(self):
        # (camelCase name, type, default, is_list)
        return [
            ("basesPerPartition", int, self.DEFAULT_NUMBER_OF_BASES_PER_SHARD, False),   # :35
            ("clientSecrets", str, None, False),                                          # :38
            ("inputPath", str, None, False),                                              # :41
            ("numReducePartitions", int, 10, False),                                      # :42
            ("outputPath", str, None, False),                                             # :46
            ("references", str, [self.PLATINUM_GENOMES_BRCA1_REFERENCES], True),         # :47
            ("sparkMaster", str, None, False),                                            # :52
            ("variantSetId", str, [GoogleGenomicsPublicData.Platinum_Genomes], True),    # :54
        ]

    def __init__(self, arguments: Sequence[str] = ()):
        parser = argparse.ArgumentParser(prog=type(self).__name__, allow_abbrev=False)
        specs = self._options()
        for name, typ, default, is_list in specs:
            flag = "--" + _kebab(name)
            if typ is bool:
                parser.add_argument(flag, dest=name, action="store_true", default=None)
            elif is_list:
                parser.add_argument(flag, dest=name, type=typ, nargs="+", default=None)
            else:
                parser.add_argument(flag, dest=name, type=typ, default=None)
        ns = parser.parse_args(list(arguments))
        for name, typ, default, is_list in specs:
            supplied = getattr(ns, name) is not None
            value = getattr(ns, name) if supplied else default
            if typ is bool and value is None:
                value = False
            setattr(self, name, Opt(_kebab(name), value, supplied))

    # GenomicsConf.scala:58-65 builds a SparkContext; here the "context" is the GPU runtime, created by the driver.
    def newSparkContext(self, className: str):
        return None

    def getPartitioner(self, references: str):
        """GenomicsConf.scala:67-69: fixed-width genomic shards (used by the synthetic/offline sources only to
        decide how many variants go into one partition)."""
        return {"references": references, "basesPerPartition": self.basesPerPartition()}


class PcaConf(GenomicsConf):
    """GenomicsConf.scala:76-101."""

    def _options(self):
        return super()._options() + [
            ("allReferences", bool, False, False),        # :77
            ("debugDatasets", bool, False, False),        # :80
            ("minAlleleFrequency", float, None, False),   # :81
            ("numPc", int, 2, False),                     # :85
            # ---- additive, GPU side ----
            ("gpuDevice", int, None, False),              # CUDA ordinal (default: LOCAL_RANK or 0)
            ("gpuDtype", str, "int8", False),             # int8 | bf16 genotype encoding
            ("synthetic", str, None, False),              # "N,V[,seed]": synthetic cohort instead of the retired API
            ("variantsPerPartition", int, 65536, False),  # rows per partition for offline/synthetic sources
            ("checkpointPath", str, None, False),         # save / resume the similarity matrix + partition watermark
            ("vcfPath", str, None, False),                # VCF file(s), comma-separated: one variant set per file
            ("callsParquetPath", str, None, False),       # Parquet file of calls rows (parquet_calls.py): RDD[Seq[Int]] at rest
            ("bedPath", str, None, False),                # PLINK 1 fileset prefix (.bed/.bim/.fam) as the variants source
            ("bedCountedAllele", str, "A1", False),       # which .bim allele is "variation": A1 (PLINK's minor) or A2
            ("saveLoadings", str, None, False),           # after computePca: write per-variant loadings + counts (.npz)
            ("projectLoadings", str, None, False),        # project this cohort onto a saved loadings file (no Gram / eigensolve)
            ("makeKingTable", str, None, False),          # --bed-path runs: write KING-robust kinship of the sample pairs here
            ("kingTableFilter", float, None, False),      # keep only the pairs with KINSHIP >= this (PLINK 2's flag names)
            ("kingCutoff", float, None, False),           # --bed-path runs: PCs of a maximal set without KINSHIP > this; the
                                                          # relatives projected onto them (PLINK 2's flag name)
            ("ldPrune", float, None, False),              # --bed-path runs: keep-first LD pruning, r2 > this within a window
            ("ldWindowKb", float, 500.0, False),          # the window of --ld-prune: same contig, positions <= this many kb apart
            ("maf", float, None, False),                  # --bed-path runs: drop variants with minor-allele frequency < this
            ("geno", float, None, False),                 # --bed-path runs: drop variants with missing-call rate > this
            ("hwe", float, None, False),                  # --bed-path runs: drop variants with exact HWE p-value < this
            ("keep", str, None, False),                   # --bed-path runs: analyse only the samples listed in this ID file
            ("remove", str, None, False),                 # --bed-path runs: leave out the samples listed in this ID file
            ("mind", float, None, False),                 # --bed-path runs: drop samples with missing-call rate > this
            ("grm", bool, False, False),                  # --bed-path runs: PCs of the variance-standardized relationship
                                                          # matrix of allele dosages (PLINK 2 / GCTA / EIGENSOFT) instead of S
            ("makeRel", bool, False, False),              # with --grm and --output-path P: write P.rel.bin and P.rel.id
            ("saveGrmLoadings", str, None, False),        # with --grm: write per-variant GRM loadings and z tables (.npz)
            ("pheno", str, None, False),                  # with --glm: the phenotype file (PLINK 2's flag names below)
            ("phenoName", str, None, False),              # with --glm: the --pheno column to test (default: the first)
            ("covar", str, None, False),                  # with --glm: a file of covariates, all used beside the PCs
            ("glm", bool, False, False),                  # --bed-path runs: linear association tests with the PCs as
                                                          # covariates, written to P.<PHENO>.glm.linear
            ("glmLogistic", bool, False, False),          # with --glm: a case/control phenotype (1 control, 2 case) by
                                                          # logistic regression, written to P.<PHENO>.glm.logistic
            ("glmFirth", str, None, False),               # with --glm --glm-logistic: fallback (Firth regression where
                                                          # the plain fit fails; P.<PHENO>.glm.logistic.hybrid) or
                                                          # always (P.<PHENO>.glm.firth)
        ]
