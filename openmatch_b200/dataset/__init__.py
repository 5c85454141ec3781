from .data_collator import DRInferenceCollator, QPCollator
from .inference_dataset import InferenceDataset, JsonlDataset, PretokenizedDataset, TsvDataset, write_ragged_store
from .train_dataset import DRTrainDataset

__all__ = ["DRInferenceCollator", "QPCollator", "InferenceDataset", "JsonlDataset", "TsvDataset",
           "PretokenizedDataset", "DRTrainDataset", "write_ragged_store"]
