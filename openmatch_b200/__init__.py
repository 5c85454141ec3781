"""openmatch_b200 — H100-native (sm_90a) dense-retrieval hot path behind OpenMatch's own entry points.

Host side mirrors the reference package layout (``modeling``, ``retriever``, ``loss``, ``driver``,
``arguments``, ``utils``); the three hot steps run in hand-written CUDA behind the C ABI declared in
``include/openmatch_b200.h`` (``csrc/``).  No CPU fallback exists in this package.
"""
__version__ = "0.1.0"
