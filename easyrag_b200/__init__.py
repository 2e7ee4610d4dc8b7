"""easyrag_b200 -- H100-native coarse ranking (dense + BM25 + RRF) behind EasyRAG's retriever API."""
__version__ = "0.1.0"
