"""CPU oracle for the dense-retrieval hot path (encode -> flat inner-product top-k -> contrastive loss).

TEST INFRASTRUCTURE ONLY.  Nothing under ``openmatch_b200/`` imports this package: the product path is
CUDA-only and fails loudly when the extension is missing.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it, and only as the checker or as the
timed CPU baseline.

Pinning status (see DESIGN.md "Oracle"):
  * encoder / pooling / head / normalise and the contrastive loss are pinned against the reference's own
    Python code (``/root/reference/src/openmatch``) executed in the build container;
    ``tests/golden/make_golden.py`` is the generating script and ``tests/golden/*.npz`` the committed vectors.
  * the flat inner-product index restates faiss ``IndexFlatIP`` (faiss is an undeclared, un-vendored,
    un-installed dependency of the reference; the reference ships no test or golden vector for it), so for
    the search step parity is anchored on the reference's call sites only: **parity unpinned** w.r.t. faiss.
"""
from .flat_index import (  # noqa: F401
    FlatIPIndex, flat_ip_search, merge_topk, merge_retrieval_results_by_score,
)
from .loss import contrastive_loss, contrastive_loss_fwd_bwd  # noqa: F401
from .encoder import (  # noqa: F401
    bert_encode, t5_encode, pool_head_normalize, encode_reps, t5_relative_position_bucket, EncoderSpec,
)
