from .dense_retrieval_model import DRModel, DRModelForInference, DROutput
from .linear import LinearHead
from .reranking_model import RRModel, RROutput

__all__ = ["DRModel", "DRModelForInference", "DROutput", "LinearHead", "RRModel", "RROutput"]
