"""runbookai_b200 — H100-native kNN engine behind RunbookAI's knowledge-base vector search.

Host-side mirror of the reference interface for this path (the reference is TypeScript;
Node is absent from the build image, so the mirror is Python over the same C ABI the
N-API addon binds — see INTEGRATION.md):

    VectorStore / create_vector_store   <- src/knowledge/store/vector-store.ts
    HybridRetriever / reciprocal_rank_fusion <- src/knowledge/retriever/hybrid-search.ts
    cosine_similarity / find_most_similar    <- src/knowledge/indexer/embedder.ts:168-202

`Index`, `RbkError` and `DimensionError` come from `_native`, which loads
runbookai_b200/lib/librbk_knn.so on first use and fails loudly if it has not been built
(there is no CPU or library fallback).  The numpy-only helpers (`synth`, `build`) import
without the library.
"""
__all__ = ["Index", "Group", "RbkError", "DimensionError"]


def __getattr__(name):   # PEP 562: `from runbookai_b200 import Index` loads the .so, `import runbookai_b200.synth` does not
    if name in __all__:
        from . import _native
        return getattr(_native, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
