"""H100-native compute core behind the reference's baseline-recommender API (see DESIGN.md).

Host-side mirrors of the reference's native seam:
    similarity.Compute_Similarity_Cython / Compute_Similarity   (Base/Similarity/...)
They call hand-written sm_90a kernels in libb200rec.so through the C ABI declared in include/b200rec.h.
Importing the package does not touch CUDA; the library is loaded on first use and its absence is an error.
"""
__all__ = ["similarity", "synth", "dist"]
