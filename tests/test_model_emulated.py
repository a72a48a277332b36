"""The model-level GPU parity tests (tests/test_gpu_model.py) replayed on CPU: same test bodies, same oracle, same tolerances,
with the C-ABI calls answered by tests/ops_emulator.py instead of the sm_90a kernels. What this checks is everything
*around* the kernels - the forward/backward engines, buffer layouts, flag plumbing, index plans - so that a host-side
regression shows up in the CPU suite; the kernels themselves are only ever checked by the `-m gpu` run of the same bodies.
"""
import pytest
import torch

import test_gpu_model as G
import test_gpu_optim as GO
from ops_emulator import emulated_ops


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


CPU = torch.device("cpu")
# (the golden-vector, multiple-choice and 448 px / 521-token bodies also pass through the emulator; they are left to the GPU run
# to keep this suite short - tests/test_host_orchestration.py covers the same engines at small sizes)
CASES = [
    ("test_cnn_backward", {}),                       # (224 px; forward stages and 64 px variants: tests/test_host_orchestration.py)
    ("test_transformer_forward_backward", dict(n_ex=2)),
    ("test_clipbert_end_to_end_two_clips_lse", {}),
    ("test_ragged_repeat_counts_and_eval_determinism", {}),
    ("test_pretraining_heads_mlm_itm", {}),
    ("test_forward_clips_equals_the_reference_clip_loop", {}),
]


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_gpu_model_test_body_on_emulated_ops(weights, name, kw):
    with emulated_ops() as calls:
        getattr(G, name)(cuda=CPU, weights=weights, **kw)
    assert calls["gemm"] > 0


def test_fused_adamw_gpu_test_body_on_emulated_ops():
    """tests/test_gpu_optim.py replayed on CPU: FusedAdamW's host logic (chunk planning over the flat buffers, the eight
    reference groups, clip bookkeeping, state views, operand emission flags) with cb_sumsq / cb_adamw_step restated in torch."""
    with emulated_ops():
        GO.test_fused_adamw_matches_reference_optimizer(cuda=CPU)


def test_fused_adamw_restore_round_trip_on_emulated_ops():
    """The optimizer restore test (save after two steps, step, load_state_dict, replay the step) on CPU: the plan is rebuilt
    from the restored state (ADVICE round 1: the moments / step counts of a mid-training restore were silently ignored)."""
    with emulated_ops():
        GO.test_fused_adamw_state_dict_round_trip_after_steps(cuda=CPU)

