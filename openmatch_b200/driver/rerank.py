"""``python -m openmatch.driver.rerank``: re-rank a TREC run with a cross-encoder and write the re-scored run
(reference: ``src/openmatch/driver/rerank.py``; flags as documented in ``docs/rr-msmarco-passage.md``).
``--query_path`` / ``--corpus_path`` take TSV, JSON lines or pretokenised (padded ``.npy`` / ragged ``.tokens.npy``)
stores; ``--reranking_depth`` keeps the first that many documents per query of the run."""
import logging

from ..arguments import DataArguments, InferenceArguments, ModelArguments
from ..dataset import InferenceDataset
from ..modeling import RRModel
from ..retriever import Reranker
from ..utils import load_from_trec, save_as_trec
from ._common import load_config, load_tokenizer, parse, setup_logging

logger = logging.getLogger(__name__)


def main():
    model_args, data_args, inference_args = parse((ModelArguments, DataArguments, InferenceArguments))
    setup_logging(inference_args, logger)
    logger.info("Encoding parameters %s", inference_args)
    logger.info("MODEL parameters %s", model_args)
    config = load_config(model_args)
    tokenizer = load_tokenizer(model_args, use_fast=False)
    model = RRModel.build(model_args=model_args, tokenizer=tokenizer, config=config, cache_dir=model_args.cache_dir)
    query_dataset = InferenceDataset.load(tokenizer=tokenizer, data_args=data_args, final=False, is_query=True,
                                          stream=False, cache_dir=model_args.cache_dir)
    corpus_dataset = InferenceDataset.load(tokenizer=tokenizer, data_args=data_args, final=False, is_query=False,
                                           stream=False, cache_dir=model_args.cache_dir)
    run = load_from_trec(inference_args.trec_run_path, max_len_per_q=inference_args.reranking_depth)
    reranker = Reranker(model, tokenizer, corpus_dataset, inference_args)
    result = reranker.rerank(query_dataset, run)
    if inference_args.process_index == 0:
        save_as_trec(result, inference_args.trec_save_path)


if __name__ == '__main__':
    main()
