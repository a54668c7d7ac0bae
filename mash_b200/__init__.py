"""mash_b200 -- H100-native MinHash engine behind the Mash sketch / dist / screen seams (the package keeps its name).

This package is a thin host mirror (ctypes) of the C ABI in include/mashgpu.h, which is implemented by
hand-written sm_90a CUDA in mash_b200/csrc.  There is no CPU path: loading fails loudly if
libmashgpu.so has not been built (`python -c "import __graft_entry__ as g; g.build()"`), and
Engine() fails if no CUDA device is present.
"""
from ._capi import (Engine, MashGpuError, SketchParams, DistParams, lib_path, load_library, linkage_z,
                    ALPHABET_NUCLEOTIDE, ALPHABET_PROTEIN, TAX_NONE)

__all__ = ["Engine", "MashGpuError", "SketchParams", "DistParams", "lib_path", "load_library", "linkage_z",
           "ALPHABET_NUCLEOTIDE", "ALPHABET_PROTEIN", "TAX_NONE"]
