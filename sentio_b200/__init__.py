"""sentio_b200 -- H100-native retrieve -> fuse -> rerank hot path behind chernistry/sentio's plugin surface.

Public surface (names match the reference's ``src/core/retrievers`` / ``src/core/rerankers`` modules):

    from sentio_b200.retrievers.dense  import DenseRetriever
    from sentio_b200.retrievers.sparse import BM25Retriever
    from sentio_b200.retrievers.hybrid import HybridRetriever, HybridRetrieverPlugin
    from sentio_b200.retrievers.scorers import KeywordMatchScorer, RecencyScorer, SemanticSimilarityScorer, MMRScorer
    from sentio_b200.rerankers.b200_reranker import B200Reranker
    from sentio_b200.vector_store import B200VectorStore          # QdrantClient-shaped store in HBM
    from sentio_b200.embedder import B200Embedder                  # BaseEmbedder surface, encoder forward on the GPU
    from sentio_b200.selector import create_document_selector_node # the node that follows the reranker
    from sentio_b200.pipeline import HybridPipeline, plan_layout   # batched / sharded arrays-in arrays-out path

All arithmetic runs in libsentio_b200.so (hand-written sm_90a CUDA, C ABI in include/sentio_b200.h).  Importing this
package does not touch the GPU; creating an engine without the built library or without an H100 raises.
"""
from .document import Document

__all__ = ["Document"]
__version__ = "0.1.0"
