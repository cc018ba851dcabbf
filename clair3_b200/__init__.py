"""clair3_b200 — H100 (sm_90a) implementation of Clair3's variant-calling network forward pass.

Public surface: ``clair3_b200.model.Clair3_P`` / ``Clair3_F`` (drop-in for ``clair3.model``), ``clair3_b200.dropin``
(patches the reference in place), ``clair3_b200.sharding`` (site-range sharding + weight broadcast),
``clair3_b200.synth`` (seeded synthetic checkpoints / batches) and the C-ABI in ``include/clair3_b200.h``.
"""
__version__ = "0.1.0"
