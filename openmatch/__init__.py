"""Drop-in alias: ``import openmatch`` / ``python -m openmatch.driver.build_index`` resolve to the
H100-native (sm_90a) implementation in ``openmatch_b200`` (same module, class and function names as
thunlp/OpenMatch's ``src/openmatch`` for the dense-retrieval hot path)."""
import importlib
import sys

import openmatch_b200 as _impl

__version__ = _impl.__version__
for _name in ("arguments", "utils", "loss", "modeling", "dataset", "trainer", "retriever", "driver", "mining", "embedding_store"):
    _mod = importlib.import_module("openmatch_b200." + _name)
    sys.modules[__name__ + "." + _name] = _mod
    globals()[_name] = _mod
for _sub in ("modeling.dense_retrieval_model", "modeling.linear", "modeling.reranking_model", "retriever.dense_retriever",
             "retriever.reranker", "trainer.dense_trainer", "dataset.data_collator", "dataset.inference_dataset",
             "dataset.train_dataset", "driver.build_index", "driver.retrieve", "driver.successive_retrieve",
             "driver.train_dr", "driver.build_hn", "driver.rerank"):
    sys.modules[__name__ + "." + _sub] = importlib.import_module("openmatch_b200." + _sub)
