"""spark_examples_b200 -- the H100-native VariantsPca hot path behind the reference's driver API.

Only what the path needs: `csrc/` (CUDA kernels + the C ABI of include/vpca.h, built into libvpca.so),
`native` (ctypes twin of the JNI class), and the host-side mirror of the reference interface
(`PcaConf`/`GenomicsConf`, `VariantsCommon`, `VariantsPcaDriver`, record types).
"""
from .conf import GenomicsConf, PcaConf, GoogleGenomicsPublicData            # noqa: F401
from .records import Call, CallData, Variant                                   # noqa: F401
from .variants_common import VariantsCommon                                    # noqa: F401
from .variants_pca import VariantsPcaDriver, extractCallInfo, getVariantKey    # noqa: F401

__all__ = ["GenomicsConf", "PcaConf", "GoogleGenomicsPublicData", "Call", "CallData", "Variant", "VariantsCommon",
           "VariantsPcaDriver", "extractCallInfo", "getVariantKey"]
