"""CPU oracle for the TurboPrune masked-DDP hot path.

TEST INFRASTRUCTURE ONLY.  This package is a CPU restatement (numpy for the
integer / bit-exact work, torch-CPU fp32 ops for the floating-point operators) of
the reference algorithms on the hot path named in BASELINE.json.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it, and there only as the checker / the timed CPU
baseline.  The product path (``turboprune_b200``) never imports it and fails loudly
when the CUDA library is missing.

Pinning: the reference ships no tests, golden vectors or fixtures (SURVEY.md §4), so
parity is pinned by outputs of the reference itself: ``tests/golden/make_golden.py`` and
``tests/golden/make_reference_golden.py`` import the unmodified reference modules from a
checkout of it and write the fixtures under ``tests/golden/``; ``tests/test_oracle_golden.py``
checks every oracle function against them.
"""
from .mask_ops import (  # noqa: F401
    masked_conv2d, masked_linear, masked_conv1d_k1,
    masked_conv2d_grads, masked_linear_grads,
)
from .prune import (  # noqa: F401
    sortable_key, kth_smallest, score_mag, score_grad, global_threshold, apply_threshold,
    prune_global, prune_per_layer, count_zeros, overall_sparsity_percent,
    erk_keep_probabilities, balanced_keep_probabilities, generate_densities,
)
from .train import sgd_momentum_step, allreduce_mean_mask, train_step  # noqa: F401
