"""ClipBertBaseModel.forward on CPU: the bodies of tests/test_gpu_base_model.py replayed with the C-ABI calls answered by
tests/ops_emulator.py plus the restatement of cb_attention_probs below (so the engine's base-output mode - hidden states,
attentions, the three kinds of upstream gradient, seeds - is checked on any machine), and the host-side contract: one flat
storage per head, the pending-backward count and the gradient-ready hook, standalone construction, reference state_dict keys."""
import contextlib
import math

import pytest
import torch

import dropout_ref as D
import ops_emulator
import test_gpu_base_model as G
from util import make_cfg

CPU = torch.device("cpu")


def attention_probs(qkv, text_mask, lse, probs, nseq, l, lt, heads, p, seed):
    """cb_attention_probs: exp(S - lse) from the GIVEN lse (as the kernel does), times the forward's dropout multipliers (the
    emulator's restated masks, with the bound device word folded into the seed)."""
    hd = qkv.shape[1] // (3 * heads)
    q, k = (x.double().reshape(nseq, l, heads, hd).permute(0, 2, 1, 3) for x in qkv.view(nseq, l, 3, heads * hd).unbind(2)[:2])
    madd = torch.cat([(text_mask[:, :lt] == 0).double() * -10000.0, torch.zeros(nseq, l - lt, dtype=torch.float64)], dim=1)
    pr = torch.exp(q @ k.transpose(-1, -2) / math.sqrt(hd) + madd[:, None, None, :] - lse.double()[..., None])
    mult = ops_emulator._drop_mult(p, seed, D.attention_index(nseq, heads, l))
    if mult is not None:
        pr = pr * mult.double()
    probs.copy_(pr)


@contextlib.contextmanager
def emulated_ops():
    """ops_emulator.emulated_ops with ops.attention_probs answered (and counted) by the restatement above."""
    from clipbert_b200 import ops
    with ops_emulator.emulated_ops() as calls:
        saved = ops.attention_probs
        calls["attention_probs"] = 0

        def counted(*a, **k):
            calls["attention_probs"] += 1
            return attention_probs(*a, **k)
        ops.attention_probs = counted
        try:
            yield calls
        finally:
            ops.attention_probs = saved


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def test_outputs_and_hidden_states_equal_the_oracle_on_emulated_ops(weights):
    with emulated_ops() as calls:
        G.test_base_model_against_oracle(cuda=CPU, weights=weights, size="224px")
    assert calls["attention_probs"] == 12 and calls["attention_fwd"] == 12


def test_gradients_match_oracle_autograd_on_emulated_ops(weights):
    with emulated_ops() as calls:
        G.test_base_model_gradients(cuda=CPU, weights=weights, nseq=2, lt=12, gh=2)
    assert calls["attention_bwd"] == 12


def test_train_mode_attentions_use_the_forward_masks_on_emulated_ops(weights):
    with emulated_ops():
        G.test_train_mode_attentions_carry_the_forward_dropout_mask(cuda=CPU, weights=weights)


def test_heads_ignore_the_output_flags_on_emulated_ops(weights):
    with emulated_ops() as calls:
        G.test_heads_ignore_the_output_flags(cuda=CPU, weights=weights)
    assert calls["attention_probs"] == 0 and calls["attention_fwd"] == 4 * 12


def test_bert_inside_a_clipbert_uses_the_heads_flat_storage(weights):
    """model.transformer.bert(...) runs the head's engine: no second flat storage, gradients in the head's flat buffer (what
    FusedAdamW, allreduce_grads and no_sync read), the pending-backward count and the gradient-ready hook see the pass."""
    import clipbert_b200 as cb
    from oracle import synth
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = cb.ClipBert(cfg, detectron2_model_cfg="R-50-grid.yaml", transformer_cls=cb.ClipBertForVideoTextRetrieval)
    model.load_state_dict(weights)
    tr = model.transformer
    assert tr.bert._engine is tr and set(tr.state_dict()) == {k[len("transformer."):] for k in weights if k.startswith("transformer.")}
    fired = []
    tr._grad_ready_hook = lambda g: fired.append(float(g.abs().sum()))
    ids, mask = synth.synth_text(2, 10, seed=5)
    grid = torch.randn(2, 1, 2, 2, 768, generator=torch.Generator().manual_seed(6)).to(torch.bfloat16).requires_grad_(True)
    with emulated_ops():
        seq, pooled = tr.bert(ids, grid, mask)
        flat = tr._flat
        assert tr._pending_backward == 1 and seq.shape == (2, 14, 768) and pooled.shape == (2, 768)
        (seq.float().sum() + pooled.float().sum()).backward()
    assert tr._flat is flat and tr._pending_backward == 0 and len(fired) == 1 and fired[0] > 0
    lo, hi = flat.grad.data_ptr(), flat.grad.data_ptr() + 4 * flat.grad.numel()
    for p in tr.bert.parameters():
        assert lo <= p.grad.data_ptr() < hi
    assert float(tr.bert.encoder.layer[0].attention.self.query.weight.grad.abs().sum()) > 0
    assert float(tr.classifier[0].weight.grad.abs().sum()) == 0          # the head was not run
    assert grid.grad is not None and float(grid.grad.float().abs().sum()) > 0


def test_standalone_base_model_state_dict_and_initialisation(weights):
    """A ClipBertBaseModel of its own: reference state_dict keys (it loads a reference-keyed dict strictly), BertPreTrainedModel
    init (N(0, 0.02) Linear / Embedding weights, zero biases, LayerNorm (1, 0)), its own flat storage, flags from the config."""
    import clipbert_b200 as cb
    from oracle import synth
    torch.manual_seed(3)
    m = cb.ClipBertBaseModel(make_cfg())
    assert m.output_hidden_states is False and m.output_attentions is False
    keys = {k[len("transformer.bert."):] for k in weights if k.startswith("transformer.bert.")}
    assert set(m.state_dict()) == keys and "_engine" not in dict(m.named_modules())
    w = m.encoder.layer[3].intermediate.dense.weight.detach()
    assert abs(float(w.std()) - 0.02) < 1e-3 and float(m.encoder.layer[3].intermediate.dense.bias.abs().max()) == 0
    assert abs(float(m.embeddings.word_embeddings.weight.std()) - 0.02) < 1e-3
    assert bool((m.pooler.dense.bias == 0).all()) and bool((m.embeddings.LayerNorm.weight == 1).all())
    assert bool((m.visual_embeddings.LayerNorm.bias == 0).all())
    ids, mask = synth.synth_text(2, 6, seed=8)
    grid = torch.randn(2, 1, 2, 2, 768)
    with emulated_ops():
        with torch.no_grad():
            seq, pooled = m(ids, grid, mask)
        assert m._engine._flat is not None and m._engine.bert is m
        m.load_state_dict({k: weights["transformer.bert." + k] for k in keys})
        with torch.no_grad():
            seq2, _ = m(ids, grid, mask)
    assert seq.shape == seq2.shape == (2, 10, 768) and not torch.equal(seq, seq2)     # the loaded weights are used


def test_reference_import_path_resolves_to_the_base_model():
    import sys
    import clipbert_b200 as cb
    from clipbert_b200 import compat
    saved = {k: sys.modules.get(k) for k in ("src.modeling.e2e_model", "src.modeling.modeling", "src.modeling.grid_feat")}
    try:
        compat.alias_reference_modules()
        from src.modeling.modeling import ClipBertBaseModel
        assert ClipBertBaseModel is cb.ClipBertBaseModel and ClipBertBaseModel.forward is not torch.nn.Module.forward
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
