from .dense_retriever import FaissRetriever, Retriever, SuccessiveRetriever
from .reranker import Reranker

__all__ = ["Retriever", "SuccessiveRetriever", "FaissRetriever", "Reranker"]
