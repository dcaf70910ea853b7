"""nvmolkit_b200 — the batched-molecule hot path of nvMolKit, rebuilt for H100 (sm_90a).

Module names and call signatures mirror ``nvmolkit.{fingerprints, similarity, clustering, embedMolecules,
mmffOptimization, uffOptimization, types}``; the compute is hand-written CUDA behind the C-ABI in
``include/b200mol.h`` (``nvmolkit_b200/lib/libb200mol.so``). No CPU fallback exists.
"""

__version__ = "0.1.0"
