"""Module hooks on ClipBertBaseModel on the CPU: the taps of tests/test_gpu_transformer_hooks.py's oracle restatement pinned to the
oracle, and its module runners replayed with the C-ABI calls answered by tests/ops_emulator.py (with the attention-map
restatements of the earlier emulated tests). Planted faults in the node chain must fail."""
import contextlib

import pytest
import torch

import test_gpu_attention_retained_grads as RG
import test_gpu_transformer_hooks as TH
import test_layerwise_autograd_emulated as LWE

CPU = torch.device("cpu")


@contextlib.contextmanager
def emulated():
    """The layerwise replays' emulated ops, with the word-vector entry points restated on the emulator's text-embedding ops: the
    vectors as a table indexed by row (word[r] = vec[r]), and the scatter as an index_add into the table."""
    import ops_emulator
    from clipbert_b200 import ops
    with LWE.emulated_ops() as calls:
        saved = {n: getattr(ops, n) for n in ("embed_text_fwd_vectors", "embed_text_bwd_vectors", "embed_word_scatter")}

        def fwd(vec, pos, typ, gamma, beta, out, stats, nseq, lt, l, eps, p, seed):
            rows = torch.arange(nseq * lt).view(nseq, lt)
            ops_emulator.embed_text_fwd(rows, vec.contiguous(), pos, typ, gamma, beta, out, stats, nseq, lt, l, eps, p, seed)

        def bwd(dh, vec, pos, typ, gamma, stats, dvec, dpos, dtyp, dgamma, dbeta, nseq, lt, l, p, seed):
            rows = torch.arange(nseq * lt).view(nseq, lt)
            dvec.zero_()
            ops_emulator.embed_text_bwd(dh, rows, vec.contiguous(), pos, typ, gamma, stats, dvec, dpos, dtyp, dgamma, dbeta, nseq, lt,
                                        l, p, seed)
        ops.embed_text_fwd_vectors, ops.embed_text_bwd_vectors = fwd, bwd
        ops.embed_word_scatter = lambda ids, dvec, dword: dword.index_add_(0, ids.reshape(-1), dvec)
        try:
            yield calls
        finally:
            for n, f in saved.items():
                setattr(ops, n, f)


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.full_state_dict(42)


def test_restatement_with_identity_taps_is_the_oracle(weights):
    from oracle import clipbert_ref as R
    grid, ids, mask, L, g = RG._inputs("224px", 1)
    mult = {i: (torch.rand(ids.shape[0], 12, L, L, generator=g) > 0.1).float() / 0.9 for i in range(12)}

    def drop(site, layer, x):
        return x * mult[layer] if site == "attn_probs" else x
    seq, pooled = R.clipbert_base_model(ids, grid, mask, weights, drop=drop)
    rec, tap = TH.ref_recorder()
    seq_t, pooled_t = TH.ref_bert(ids, grid, mask, weights, mult, tap)
    assert torch.allclose(seq_t, seq, rtol=1e-5, atol=1e-5) and torch.allclose(pooled_t, pooled, rtol=1e-5, atol=1e-5)
    sites = [s for s, _ in TH.site_modules(_bert_for_names(weights))]
    assert all(TH.ref_site(s) in rec for s in sites) and len(sites) == 5 + 12 * 6


def _bert_for_names(weights):
    import clipbert_b200 as cb
    return cb.ClipBertBaseModel(TH.make_cfg())


def test_every_site_against_oracle_on_emulated_ops(weights):
    with emulated():
        TH.run_sites_against_oracle(CPU, weights, "cpu")


def test_every_site_with_differentiable_maps_on_emulated_ops(weights):
    with emulated():
        TH.run_sites_against_oracle(CPU, weights, "cpu", diff_attn=True)


@pytest.mark.parametrize("which", ["bert", "retrieval", "ragged"])
def test_observe_only_hooks_keep_the_bits_on_emulated_ops(weights, which):
    with emulated():
        TH.run_bits_observe_only(CPU, weights, "cpu", which)


@pytest.mark.parametrize("which", ["tokens", "heads", "patch", "word", "grad"])
def test_interventions_on_emulated_ops(weights, which):
    with emulated():
        TH.run_interventions(CPU, weights, "cpu", which)


@pytest.mark.parametrize("site", ["embeddings", "word_embeddings"])
def test_integrated_gradients_on_emulated_ops(weights, site):
    with emulated():
        TH.run_integrated_gradients(CPU, weights, "cpu", steps=8, site=site)


@pytest.mark.parametrize("cls_name,cfg", TH.HEADS, ids=[h[0] for h in TH.HEADS])
def test_head_hooks_on_emulated_ops(weights, cls_name, cfg):
    with emulated():
        TH.run_head_hooks(CPU, weights, "cpu", cls_name, cfg)


def test_semantics_on_emulated_ops(weights):
    with emulated() as calls:
        TH.run_semantics(CPU, weights, "cpu", launches=calls)


def test_refusals_on_emulated_ops(weights):
    with emulated():
        TH.run_refusals(CPU, weights)


# ------------------------------------------------------------------------------------------------ planted faults
def test_fault_residual_owner_seen_as_not_running_breaks_the_bits(weights, monkeypatch):
    """The residual's two bf16 contributions summed by autograd (rounded twice) instead of handed over."""
    from clipbert_b200 import modeling
    runs = modeling._engine_runs

    def partner_never_runs(node, captured):      # the residual's owner (_SelfNode, _InterNode) seen as not running
        return runs(node, captured) and type(node).__name__ not in ("_SelfNodeBackward", "_InterNodeBackward")
    monkeypatch.setattr(modeling, "_engine_runs", partner_never_runs)
    with emulated():
        with pytest.raises(AssertionError):
            TH.run_bits_observe_only(CPU, weights, "cpu", "bert")


def test_fault_handover_never_taken_fails_the_oracle(weights, monkeypatch):
    """The residual handed over but never added by the receiving node."""
    from clipbert_b200 import modeling
    orig = modeling._BertPass.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        self.handover = _Forgetful()
    monkeypatch.setattr(modeling._BertPass, "__init__", init)
    with emulated():
        with pytest.raises(AssertionError):
            TH.run_sites_against_oracle(CPU, weights, "cpu")


class _Forgetful(dict):
    def pop(self, key, default=None):
        if isinstance(key, tuple):
            dict.pop(self, key, None)
            return default
        return dict.pop(self, key, default)


def test_fault_wrong_dropout_seed_fails_the_oracle(weights, monkeypatch):
    from clipbert_b200 import modeling
    monkeypatch.setattr(modeling, "_layer_seed", lambda ps, i: ps.st["seed"] + 16 * (i + 1) + 16)
    with emulated():
        with pytest.raises(AssertionError):
            TH.run_sites_against_oracle(CPU, weights, "cpu")


def test_fault_replaced_context_in_the_self_attention_piece_fails_the_oracle(weights, monkeypatch):
    """The attention backward fed the context a hook replaced instead of the forward's own O (its D = rowsum(dO o O) term)."""
    from clipbert_b200 import modeling
    orig = modeling._ClipBertHeadModel._self_attention_backward

    def wrong(self, st, i, ly, *args, **kw):
        ly = dict(ly, ctx=ly["ctx"] * TH._head_scale().to(ly["ctx"].dtype)) if i == 5 else ly
        return orig(self, st, i, ly, *args, **kw)
    monkeypatch.setattr(modeling._ClipBertHeadModel, "_self_attention_backward", wrong)
    with emulated():
        with pytest.raises(AssertionError):
            TH.run_interventions(CPU, weights, "cpu", "heads")
