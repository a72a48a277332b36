"""Cross-modal transformer half of ClipBERT on H100.

Mirrors the reference classes in ``src/modeling/modeling.py`` / ``src/modeling/transformers.py``
(ClipBertBaseModel, ClipBertForVideoTextRetrieval, ClipBertForSequenceClassification,
ClipBertForMultipleChoice, ClipBertForPreTraining): same constructor (a BertConfig-like object),
same forward signatures and return dicts, same state_dict keys (SURVEY.md App. B). The torch.nn
modules below are parameter containers whose ``forward`` runs only on the module path: when a hook is registered on bert or a
module below it, bert(...) and the heads call them (_BertPass), each running its part of the engine; so does bert(...) with
layerwise_autograd on. All arithmetic is the hand-written sm_90a kernels behind libclipbert_sm90.so:

  embeddings     cb_embed_text_fwd / cb_embed_visual_fwd (gather + sum + LN + dropout; the visual
                 kernel also fuses the frame mean, the row/col/type adds, repeat_tensor_rows and
                 the [text ; visual] concat by writing at sequence offset Lt)
  encoder layer  cb_gemm (QKV fused N=2304, +bias) -> cb_attention_fwd -> cb_gemm (+bias, dropout,
                 +residual) -> cb_layernorm_fwd -> cb_gemm (+bias, GELU, pre-activation stash) ->
                 cb_gemm (+bias, dropout, +residual) -> cb_layernorm_fwd
  pooler / head  cb_gemm (strided [CLS] rows, +bias, tanh) -> cb_dropout -> cb_gemm (ReLU) -> cb_gemm
  backward       mirror image; dgrad = cb_gemm NN straight from the forward weight layout, wgrad =
                 cb_gemm WGRAD accumulating fp32 into the flat gradient buffer, activation
                 derivatives and dropout masks fused into the dgrad / LayerNorm-backward epilogues.
"""
import contextlib
import weakref

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .params import FlatGroup

_SEED_STRIDE = 0x9E3779B97F4A7C15


def _cfg(config, name, default=None):
    if isinstance(config, dict):
        return config.get(name, default)
    return getattr(config, name, default)


# ----------------------------------------------------------------------------------------------------
# parameter containers (names = reference attribute names => identical state_dict keys)
# ----------------------------------------------------------------------------------------------------
class BertWordEmbeddings(nn.Embedding):
    """BertEmbeddings.word_embeddings: on the module path (a hook on it) input_ids -> word[input_ids], fp32 (B', Lt, 768)."""

    def forward(self, input_ids):
        return _bert_pass(self).word(self, input_ids)


class BertEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.word_embeddings = BertWordEmbeddings(_cfg(config, "vocab_size"), h, padding_idx=_cfg(config, "pad_token_id", 0))
        self.position_embeddings = nn.Embedding(_cfg(config, "max_position_embeddings"), h)
        self.token_type_embeddings = nn.Embedding(_cfg(config, "type_vocab_size"), h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))

    def forward(self, input_ids):
        return _bert_pass(self).text(self, input_ids)


class VisualInputEmbedding(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.position_embeddings = nn.Embedding(_cfg(config, "max_position_embeddings"), h)   # unused (modeling.py:97)
        self.row_position_embeddings = nn.Embedding(_cfg(config, "max_grid_row_position_embeddings"), h)
        self.col_position_embeddings = nn.Embedding(_cfg(config, "max_grid_col_position_embeddings"), h)
        self.token_type_embeddings = nn.Embedding(1, h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))

    def forward(self, grid):
        return _bert_pass(self).visual(self, grid)


class BertSelfAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.query, self.key, self.value = nn.Linear(h, h), nn.Linear(h, h), nn.Linear(h, h)

    def forward(self, hidden_states, attention_mask=None, head_mask=None):
        return _bert_pass(self).self_attention(self, hidden_states, attention_mask, head_mask)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.dense = nn.Linear(h, h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))

    def forward(self, hidden_states, input_tensor):
        return _bert_pass(self).self_output(self, hidden_states, input_tensor)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)

    def forward(self, hidden_states, attention_mask=None, head_mask=None):
        return _bert_pass(self).attention(self, hidden_states, attention_mask, head_mask)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(_cfg(config, "hidden_size"), _cfg(config, "intermediate_size"))

    def forward(self, hidden_states):
        return _bert_pass(self).intermediate(self, hidden_states)


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(_cfg(config, "intermediate_size"), _cfg(config, "hidden_size"))
        self.LayerNorm = nn.LayerNorm(_cfg(config, "hidden_size"), eps=_cfg(config, "layer_norm_eps"))

    def forward(self, hidden_states, input_tensor):
        return _bert_pass(self).output(self, hidden_states, input_tensor)


class BertLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)

    def forward(self, hidden_states, attention_mask=None, head_mask=None):
        return _bert_pass(self).layer(self, hidden_states, attention_mask, head_mask)


class BertEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layer = nn.ModuleList([BertLayer(config) for _ in range(_cfg(config, "num_hidden_layers"))])

    def forward(self, hidden_states, attention_mask=None, head_mask=None):
        return _bert_pass(self).encoder(self, hidden_states, attention_mask, head_mask)


class BertPooler(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.dense = nn.Linear(h, h)

    def forward(self, hidden_states):
        return _bert_pass(self).pooler(self, hidden_states)


class ClipBertBaseModel(nn.Module):
    """src/modeling/modeling.py:156-238: embeddings + 12 BertLayers + pooler, the building block every head calls as
    ``self.bert(...)``.

    ``forward(text_input_ids, visual_inputs, attention_mask)`` returns ``(sequence_output, pooled_output)``, then
    ``(all_hidden_states,)`` and ``(all_attentions,)`` when ``config.output_hidden_states`` / ``config.output_attentions``
    are set (read at construction, as BertEncoder does; missing = False). ``visual_inputs`` is (B', T, h, w, 768) with one
    row per text example (repeat_tensor_rows already applied).

    Inside a head (``head.bert``) the call runs the head's engine: the parameters are views into the head's flat storage and
    their gradients land in its flat gradient buffer. Constructed on its own, the model gets an engine and flat storage of
    its own and initialises its weights as BertPreTrainedModel.init_weights does.

    Dtypes: sequence_output, pooled_output and the 13 hidden states are bf16 - the engine's own activation buffers, no copy
    (the reference's amp-O2 runs hand out fp16 here). The attentions are fp32 (B', heads, L, L), one per layer, the
    post-dropout probabilities. Autograd flows from sequence_output, pooled_output and every hidden state into every
    parameter and into ``visual_inputs``.

    ``model.differentiable_attentions = True`` (default False; also on ``head.bert``) makes the attentions of a pass that
    records autograd differentiable too, as the reference's are: a loss on ``attentions[layer]`` (attention supervision,
    distillation of a teacher's maps, entropy penalties) then trains every parameter below that layer and ``visual_inputs``,
    through cb_attention_probs_bwd (include/clipbert_b200.h). A pass whose loss does not use the attentions costs and
    computes exactly what it does with the switch off. With the default the attentions are returned non-differentiable.

    ``t.retain_grad()`` on a returned tensor gives, after ``backward()``, the ``.grad`` the reference's tensor holds (the HF
    idiom of gradient-based attribution: attention x gradient relevance, Grad-SAM, gradient x input on the hidden states):
    ``attentions[l].grad`` (switch on) is the loss's direct term plus dO V^T per head, the term from the context product
    (cb_attention_dprobs: dO = d loss / d context of layer l, V its bf16 value block; at every position, dropped ones
    included); ``hidden_states[k].grad`` is the full gradient at the input of layer k, and ``sequence_output.grad`` (the
    same tensor as hidden_states[12] in the reference) the full top gradient, pooler path included; ``pooled_output.grad``
    is its direct term, which is its full gradient. A pass with nothing retained issues the same launches as without.

    By default the whole pass is one autograd node: a tensor hook on a map or hidden state fires before that node runs and sees
    only the loss's direct term, and ``torch.autograd.grad(score, attentions)`` (or hidden states) returns only that term.
    ``model.layerwise_autograd = True`` (default False; also on ``head.bert``) runs a pass that records autograd through the
    modules, as a hook does (below), so that it is a chain of nodes - the embeddings, one node per encoder layer
    (two when the maps are differentiable: A_k, hidden_states[k] -> attentions[k], and C_k, (hidden_states[k], attentions[k])
    -> hidden_states[k + 1], the reference's dataflow) and the pooler - with sequence_output the same tensor as
    hidden_states[12]. With a hook set as well, the hooks decide where the chain splits. Tensor hooks, ``torch.autograd.grad``,
    ``retain_grad()`` and ``backward(inputs=...)`` on any map or hidden state then follow torch's semantics, and a hook that
    rewrites a map's gradient changes every gradient below that layer. Parameter gradients too: a node writes them only when
    the backward accumulates into the parameters (``autograd.grad`` leaves the flat gradient buffer as it was), and
    ``retain_graph=True`` allows a second backward. The forward issues the launches of the default; so does the backward of a
    layer whose map is not differentiable. Refused together with the overlapped data-parallel exchange
    (``enable_overlapped_allreduce``): the switch is for analysis, not training.

    A hook on this model or a module below it (or a global module hook) runs the pass through the modules - embeddings,
    visual_embeddings, encoder, each layer's attention (self, output), intermediate and output, pooler - so torch's hooks on them
    fire, and a forward hook or pre-hook may replace what they return or receive. The backward is a chain of nodes split at the
    hooked modules. INTEGRATION.md lists what each module hands to its hooks and the hooks that are refused.

    ``model.recompute_activations = True`` (default False; also on ``head.bert``) trades compute for activation memory, as
    wrapping each BertLayer in ``torch.utils.checkpoint`` does on the reference: a pass that records autograd keeps only each
    encoder layer's input hidden state, and the backward re-runs the layer's forward (same launches, seeds and dropout word, so
    the same masks, under CUDA-graph replay too) just before that layer's backward. The gradients are bit-identical to the
    switch off in deterministic mode. Refused together with ``differentiable_attentions``, ``layerwise_autograd`` and module
    hooks, whose backward reads every layer's activations as saved tensors.
    """

    differentiable_attentions = False
    layerwise_autograd = False
    recompute_activations = False

    def __init__(self, config, _engine=None):
        super().__init__()
        self.config = config
        self.embeddings = BertEmbeddings(config)
        self.visual_embeddings = VisualInputEmbedding(config)
        self.encoder = BertEncoder(config)
        self.pooler = BertPooler(config)
        self.output_hidden_states = bool(_cfg(config, "output_hidden_states", False))
        self.output_attentions = bool(_cfg(config, "output_attentions", False))
        if _engine is None:
            _init_bert_weights(self, _cfg(config, "initializer_range", 0.02))
            _engine = _BaseModelEngine(config, self)
        # a back-reference, not a submodule: state_dict keys stay the reference's, and a head keeps one flat storage
        self.__dict__["_engine"] = _engine

    def forward(self, text_input_ids, visual_inputs, attention_mask):
        eng = self._engine
        ps = _BERT_PASSES[-1] if _BERT_PASSES and _BERT_PASSES[-1].awaits(eng) else None
        if ps is None:
            ps, records = eng._base_pass(visual_inputs)
            if ps is None:
                return eng._run_base(text_input_ids, visual_inputs, attention_mask, self.output_hidden_states, self.output_attentions,
                                     self.differentiable_attentions, records)
            with ps:
                return ps.base(text_input_ids, visual_inputs, attention_mask)
        return ps.base(text_input_ids, visual_inputs, attention_mask)


def _require_cuda(t):
    assert t.is_cuda, "ClipBERT transformer runs on CUDA only (no CPU fallback)"


def get_random_sample_indices(seq_len, num_samples=100, device=torch.device("cpu")):
    """src/modeling/modeling.py:15-34: sorted indices of a sample without replacement, drawn from numpy's global
    generator exactly as the reference does (np.random.seed reproduces its choice); all indices if num_samples >= seq_len."""
    import numpy as np
    if num_samples >= seq_len:
        sample_indices = np.arange(seq_len)
    else:
        sample_indices = np.sort(np.random.choice(seq_len, size=num_samples, replace=False))
    return torch.from_numpy(sample_indices).long().to(device)


def _init_bert_weights(module, std):
    """BertPreTrainedModel._init_weights (src/modeling/transformers.py:559-570)."""
    for m in module.modules():
        if isinstance(m, (nn.Linear, nn.Embedding)):
            m.weight.data.normal_(mean=0.0, std=std)
        elif isinstance(m, nn.LayerNorm):
            m.bias.data.zero_()
            m.weight.data.fill_(1.0)
        if isinstance(m, nn.Linear) and m.bias is not None:
            m.bias.data.zero_()


class _Lin:
    """Packed views of one (possibly fused / zero-padded) linear layer."""
    __slots__ = ("w", "b", "gw", "gb", "n", "k")


class _TransformerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, grid, anchor, ids, mask, repeat):
        out, stash = module._forward_impl(ids, grid, mask, repeat, need_backward=True)
        module._pending_backward += 1
        ctx.module, ctx.stash = module, stash
        ctx.grid_needs_grad = grid.requires_grad
        return out

    @staticmethod
    def backward(ctx, *douts):
        stash, ctx.stash = ctx.stash, None
        m = ctx.module
        dgrid = m._backward_impl(stash, douts if len(douts) > 1 else douts[0], ctx.grid_needs_grad)
        m._backward_done()
        return None, dgrid, None, None, None, None


class _BaseModelFn(torch.autograd.Function):
    """ClipBertBaseModel.forward as one autograd node: outputs (sequence_output, pooled_output, *hidden_states, *attentions)."""

    @staticmethod
    def forward(ctx, module, grid, anchor, ids, mask, flags):
        (seq, pooled, hidden, attn), stash = module._forward_impl(ids, grid, mask, (1, None, None), need_backward=True, base=flags)
        module._pending_backward += 1
        ctx.module, ctx.stash = module, stash
        ctx.grid_needs_grad = grid.requires_grad
        ctx.n_hidden = len(hidden)
        if not flags[2]:                        # ClipBertBaseModel.differentiable_attentions
            ctx.mark_non_differentiable(*attn)
        ctx.set_materialize_grads(False)        # unused outputs arrive as None and cost nothing in the backward
        outs = (seq, pooled) + tuple(hidden) + tuple(attn)
        # weak: the node holding its own outputs would form a cycle (the outputs hold the node as grad_fn)
        ctx.outputs = [weakref.ref(t) for t in outs]
        return outs

    @staticmethod
    def backward(ctx, dseq, dpooled, *rest):
        stash, ctx.stash = ctx.stash, None
        m = ctx.module
        stash["base_grads"] = (dseq, dpooled, rest[:ctx.n_hidden], rest[ctx.n_hidden:])
        stash["retained"] = _BaseModelFn._retained(ctx, len(stash["layers"]))
        dgrid = m._backward_impl(stash, None, ctx.grid_needs_grad)
        m._backward_done()
        return None, dgrid, None, None, None, None

    @staticmethod
    def _retained(ctx, n_layers):
        """The outputs the caller called retain_grad() on, or None when there are none: ([tensors whose .grad is the gradient at
        the input of layer k, k = 0 .. n_layers (n_layers: the top, where sequence_output is hidden_states[n_layers])],
        [attentions[i] or None]). torch's retain hooks run before this node's backward, so each .grad holds the loss's direct
        term on that output, if any, when the engine reads it."""
        outs = [r() for r in ctx.outputs]
        outs = [t if t is not None and t.retains_grad else None for t in outs]
        if all(t is None for t in outs):
            return None
        hidden, attn = outs[2:2 + ctx.n_hidden], outs[2 + ctx.n_hidden:]
        at_input = [[] for _ in range(n_layers + 1)]
        for k, t in enumerate(hidden):
            if t is not None:
                at_input[k].append(t)
        if outs[0] is not None:
            at_input[n_layers].append(outs[0])
        return at_input, (attn if any(t is not None for t in attn) else None)


_LAYER_STASH = ("x", "qkv", "ctx", "lse", "s1", "st1", "a", "u", "gel", "s2", "st2")


# ----------------------------------------------------------------------------------------------------
# module path: hooks on bert and the modules below it
# ----------------------------------------------------------------------------------------------------
_BERT_PASSES = []     # the module-path passes running (_BertPass), innermost last
_BERT_SITES = (BertEmbeddings, BertWordEmbeddings, VisualInputEmbedding, BertEncoder, BertLayer, BertAttention, BertSelfAttention, BertSelfOutput,
               BertIntermediate, BertOutput, BertPooler, ClipBertBaseModel)


def _bert_pass(module):
    """The module-path pass that is calling ``module``: bert's modules run only inside bert(...) or a head's forward."""
    if not _BERT_PASSES:
        raise RuntimeError("%s of ClipBertBaseModel runs only inside bert(...) or a head's forward (call the ClipBertBaseModel or its "
                           "head; calling its embeddings, encoder, layers or their sub-modules directly is not supported)"
                           % type(module).__name__)
    return _BERT_PASSES[-1]


def _has_hooks(mod):
    return bool(mod._forward_hooks or mod._forward_pre_hooks or mod._backward_hooks or mod._backward_pre_hooks)


def _global_hooks():
    g = torch.nn.modules.module
    return any(getattr(g, k, None) for k in ("_global_forward_hooks", "_global_forward_pre_hooks", "_global_backward_hooks",
                                             "_global_backward_pre_hooks"))


def _engine_runs(node, captured):
    """Whether the autograd engine runs ``node`` (a grad_fn; None: no gradient flows there) in the current backward. torch raises
    for a node that torch.autograd.grad() captures instead of running, and ``captured`` is the answer then: False for a parameter
    anchor (autograd.grad() does not accumulate into .grad; neither does backward(inputs=...) without the parameter), True for a
    data input whose gradient the call asks for."""
    if node is None:
        return False
    try:
        return bool(torch._C._will_engine_execute_node(node))
    except RuntimeError:
        return captured


class _BertPass:
    """One bert(...) pass on the module path (a hook on bert or a module below it, or layerwise_autograd with no hook): each module
    the forward calls runs its part of the engine here, from the tensor it was handed (the previous module's output, or what a
    hook replaced it with) to a view of the bf16 buffer it writes. A pass that records autograd runs each part as a node whose
    activations are its saved tensors: one node per encoder layer unless a sub-module of that layer is hooked, then the attention
    (or, with its self-attention or output hooked, _SelfNode + _SelfOutputNode) and the FFN (or, with intermediate or output
    hooked, _InterNode + _OutNode). split_maps (layerwise_autograd with differentiable maps): a layer with no hooked sub-module
    is two nodes, _MapNode (A_k) and _ContextNode (C_k)."""

    def __init__(self, eng, hooked, repeat=None, given=None, split_maps=False):
        self.eng, self.hooked, self.split_maps = eng, hooked, split_maps
        self.repeat = (1, None, None) if repeat is None else repeat
        self.head = repeat is not None          # a head's pass: bert(...) is called by the head and returns to it
        self.given = given                      # head: (the visual_inputs it hands to bert, the grid behind them)
        self.waiting = self.head                # the head's bert(...) call has not started yet
        self.st = None
        self.own = {}                           # id(tensor handed out) -> (tensor, the engine's [B' * L, H] rows behind it)
        self.fwd = {}                           # forward-only bookkeeping, dropped when the pass ends (it refers to outputs)
        self.handover = {}                      # backward: residual gradients handed to the node that owns the other term

    def __enter__(self):
        _BERT_PASSES.append(self)
        return self

    def __exit__(self, *exc):
        _BERT_PASSES.pop()
        self.own, self.fwd = {}, {}
        ops.dropout_offset_bind(None)

    def awaits(self, eng):
        return self.waiting and self.eng is eng

    # ---- shared helpers ------------------------------------------------------------------------------------------------
    def bind(self):
        ops.dropout_offset_bind(self.st["drop_word"])       # a hook may have run another pass in between

    def dims(self):
        nseq, _, _, _, _, lt, L = self.st["dims"]
        return nseq, lt, L, self.st["H"]

    def is_hooked(self, *mods):
        return any(m in self.hooked for m in mods)

    def give(self, t, rows):
        self.own[id(t)] = (t, rows)
        return t

    def rows(self, t, what):
        """A tensor a module was handed, as the engine's [B' * L, H] contiguous bf16 rows: the buffer behind it when it is the
        tensor the pass handed out, else a copy (a hook's replacement, any strides, bf16, fp16 or fp32)."""
        own = self.own.get(id(t))
        if own is not None and own[0] is t:
            return own[1]
        nseq, _, L, H = self.dims()
        if tuple(t.shape) != (nseq, L, H):
            raise RuntimeError("ClipBertBaseModel: %s must be a (%d, %d, %d) tensor, got %s" % (what, nseq, L, H, tuple(t.shape)))
        return t.detach().to(torch.bfloat16).reshape(nseq * L, H).contiguous()

    def dense(self, g):
        """An upstream gradient of a hidden state as the engine's [B' * L, H] contiguous bf16 operand."""
        nseq, _, L, H = self.dims()
        return g.reshape(nseq * L, H).to(torch.bfloat16).contiguous()

    def view(self, rows):
        nseq, _, L, H = self.dims()
        return rows.view(nseq, L, H)

    def layer_index(self, mod):
        return self.eng._bert_site_index()[mod]

    def check_mask(self, mod, attention_mask, head_mask):
        if attention_mask is not self.fwd.get("ext_mask"):
            raise RuntimeError("ClipBertBaseModel: the attention_mask %s received is not the extended mask of the pass: a hook that "
                               "changes the mask is not supported (the kernels read the text mask of the call)" % type(mod).__name__)
        if head_mask is not None:
            raise RuntimeError("ClipBertBaseModel: %s received a head_mask: head masks are not supported (ablate a head with a "
                               "pre-hook on attention.output that zeroes its 64 context columns)" % type(mod).__name__)

    # ---- ClipBertBaseModel ---------------------------------------------------------------------------------------------
    def base(self, ids, visual_inputs, attention_mask):
        """ClipBertBaseModel.forward through its modules (modeling.py:201-238)."""
        eng = self.eng
        bert = eng.bert
        self.waiting = False
        _require_cuda(ids)
        eng._ensure_ready(ids.device)
        src = visual_inputs
        if self.head and visual_inputs is self.given[0]:
            src = self.given[1]                 # the head's grid, repeated by the visual-embedding kernel
        else:
            self.repeat = (1, None, None)
            assert visual_inputs.shape[0] == ids.shape[0], "visual_inputs must have one row per text example"
        grid = src.detach()
        grid = (grid if grid.dtype == torch.bfloat16 else grid.to(torch.bfloat16)).contiguous()
        mask = attention_mask.to(torch.int64).contiguous()
        self.want_hidden, self.want_attn = bert.output_hidden_states, bert.output_attentions
        self.diff_attn = self.want_attn and bert.differentiable_attentions
        self.need_backward = torch.is_grad_enabled()
        self.st = eng._pass_state(ids.contiguous(), grid, mask, self.repeat, bert.training)
        self.fwd["grid"], self.fwd["grid_src"] = visual_inputs, src
        nseq, lt, L, H = self.dims()
        self.x = torch.empty(nseq * L, H, dtype=torch.bfloat16, device=ids.device)
        if self.hooked:
            t = bert.embeddings(ids)
            v = bert.visual_embeddings(visual_inputs)
            x = self.give(_JoinNode.apply(self, t, v), self.fwd.pop("x_rows"))
        else:                                   # layerwise_autograd: both embeddings as one node, in the default path's order
            x = self.give(_EmbeddingsNode.apply(self, src, bert.embeddings.word_embeddings.weight), self.x)
        ext = None
        enc_mods = [bert.encoder] + [m for ly in bert.encoder.layer for m in (ly, ly.attention, ly.attention.self)]
        if self.is_hooked(*enc_mods):         # the reference's extended additive mask, for the hooks that can see it
            full = torch.cat([mask, mask.new_ones(nseq, L - lt)], 1)
            ext = (1.0 - full[:, None, None, :].to(torch.float32)) * -10000.0
        self.fwd["ext_mask"] = ext
        enc = bert.encoder(x, ext)
        made = self.fwd.pop("encoder_out")
        if len(enc) != len(made) or any(a is not b for a, b in zip(enc[1:], made[1:])):
            raise RuntimeError("ClipBertBaseModel: a hook on bert.encoder replaced a member of its output other than [0] (the last "
                               "hidden state): not supported; replace a layer's output instead")
        pooled = bert.pooler(enc[0])
        return (enc[0], pooled) + tuple(enc[1:])

    # ---- embeddings ------------------------------------------------------------------------------------------------------
    def text(self, mod, ids):
        if ids.dtype not in (torch.int64, torch.int32) or tuple(ids.shape) != tuple(self.st["ids"].shape):
            raise RuntimeError("ClipBertBaseModel: bert.embeddings takes (%d, %d) token ids" % tuple(self.st["ids"].shape))
        ids = ids.to(torch.int64).contiguous()
        if self.is_hooked(mod.word_embeddings):
            vec = mod.word_embeddings(ids)
            return self.give(_TextVectorsNode.apply(self, vec, mod.word_embeddings.weight), self.x)
        return self.give(_TextNode.apply(self, ids, mod.word_embeddings.weight), self.x)

    def word(self, mod, ids):
        if ids.dtype not in (torch.int64, torch.int32) or tuple(ids.shape) != tuple(self.st["ids"].shape):
            raise RuntimeError("ClipBertBaseModel: bert.embeddings.word_embeddings takes (%d, %d) token ids" % tuple(self.st["ids"].shape))
        return _WordNode.apply(self, ids.to(torch.int64).contiguous(), mod.weight)

    def visual(self, mod, grid):
        st = self.st
        if grid is self.fwd["grid"]:
            g, repeat, grid = st["grid"], self.repeat, self.fwd["grid_src"]
        else:                                   # a replacement: one row per sequence, sampled as the pass samples
            nseq, nvid, T, gh, gw, _, _ = st["dims"]
            g = grid.detach()
            g = (g if g.dtype == torch.bfloat16 else g.to(torch.bfloat16)).contiguous()
            sample = st["sample"]
            shape = (nseq, T, gh * gw, 1, st["H"]) if sample is not None else (nseq, T, gh, gw, st["H"])
            if sample is not None:
                if g.shape[0] != nseq or g.dim() != 5 or g.shape[2] * g.shape[3] != sample[1] * sample[2]:
                    raise RuntimeError("ClipBertBaseModel: visual_inputs replaced with a tensor of the wrong shape %s" % (tuple(grid.shape),))
                g = g.view(nseq, T, -1, st["H"]).index_select(2, sample[0]).view(nseq, T, gh, gw, st["H"])
            elif tuple(g.shape) != (nseq, T, gh, gw, st["H"]):
                raise RuntimeError("ClipBertBaseModel: visual_inputs must be %s per sequence, got %s" % (shape, tuple(grid.shape)))
            repeat = (1, None, None)
        return self.give(_VisualNode.apply(self, grid, g, repeat, mod.LayerNorm.weight), self.x)

    # ---- encoder -----------------------------------------------------------------------------------------------------------
    def encoder(self, mod, h, attention_mask, head_mask):
        self.check_mask(mod, attention_mask, head_mask)
        hidden, attn = [], []
        for layer in mod.layer:
            if self.want_hidden:
                hidden.append(h)
            outs = layer(h, attention_mask, None)
            h = outs[0]
            if self.want_attn:
                attn.append(outs[1])
        if self.want_hidden:
            hidden.append(h)
        out = (h,) + ((tuple(hidden),) if self.want_hidden else ()) + ((tuple(attn),) if self.want_attn else ())
        self.fwd["encoder_out"] = out
        return out

    def _maps(self, outs, probs):
        return outs + ((probs,) if self.want_attn else ())

    def layer(self, mod, h, attention_mask, head_mask):
        self.check_mask(mod, attention_mask, head_mask)
        i = self.layer_index(mod)
        att = mod.attention
        if not self.is_hooked(att, att.self, att.output, mod.intermediate, mod.output):
            if self.split_maps:
                probs = _MapNode.apply(self, i, h, att.self.query.weight)
                y = _ContextNode.apply(self, i, h, probs, att.output.dense.weight)
                return self.give(y, self.fwd.pop("y_rows")), probs
            y, probs = _LayerModNode.apply(self, i, h, att.self.query.weight)
            return self._maps((self.give(y, self.fwd.pop("y_rows")),), probs)
        ao = att(h, attention_mask, None)
        a = ao[0]
        if self.is_hooked(mod.intermediate, mod.output):
            y = mod.output(mod.intermediate(a), a)
        else:
            y = self.give(_FfnNode.apply(self, i, a, mod.intermediate.dense.weight), self.fwd.pop("y_rows"))
        return (y,) + tuple(ao[1:])

    def attention(self, mod, h, attention_mask, head_mask):
        self.check_mask(mod, attention_mask, head_mask)
        i = self.layer_index(mod)
        if self.is_hooked(mod.self, mod.output):
            so = mod.self(h, attention_mask, None)
            return (mod.output(so[0], h),) + tuple(so[1:])
        a, probs = _AttentionNode.apply(self, i, h, mod.self.query.weight)
        return self._maps((self.give(a, self.fwd.pop("a_rows")),), probs)

    def self_attention(self, mod, h, attention_mask, head_mask):
        self.check_mask(mod, attention_mask, head_mask)
        i = self.layer_index(mod)
        ctx, probs = _SelfNode.apply(self, i, h, mod.query.weight)
        self.fwd[("self", i)] = (h, ctx.grad_fn)
        return self._maps((self.give(ctx, self.fwd.pop("ctx_rows")),), probs)

    def self_output(self, mod, ctx, h):
        i = self.layer_index(mod)
        h_self, node = self.fwd.pop(("self", i), (None, None))
        partner = node if (h_self is h and node is not None) else None
        a = _SelfOutputNode.apply(self, i, ctx, h, mod.dense.weight, partner)
        return self.give(a, self.fwd.pop("a_rows"))

    def intermediate(self, mod, a):
        i = self.layer_index(mod)
        gel = _InterNode.apply(self, i, a, mod.dense.weight)
        self.fwd[("inter", i)] = (a, gel.grad_fn)
        return gel

    def output(self, mod, gel, a):
        i = self.layer_index(mod)
        a_inter, node = self.fwd.pop(("inter", i), (None, None))
        partner = node if (a_inter is a and node is not None) else None
        y = _OutNode.apply(self, i, gel, a, mod.dense.weight, partner)
        return self.give(y, self.fwd.pop("y_rows"))

    # ---- pooler and head -----------------------------------------------------------------------------------------------
    def split_head(self):
        """Whether the head's part runs as a node of its own after the pooler (pooled_output visible to a hook), rather than
        together with the pooler's backward (its tanh' fused into the head's dgrad epilogue, as on the default path)."""
        return self.is_hooked(self.eng.bert, self.eng.bert.pooler)

    def pooler(self, mod, h):
        self.fwd["seq"] = h
        if self.head and not self.split_head():
            x = self.rows(h, "the input of bert.pooler")
            self.fwd["seq_rows"] = x
            self.bind()
            return self.eng._pooler_fwd(self.st, x)           # the head's node runs the pooler's backward
        return _PoolerModNode.apply(self, h, mod.dense.weight)

    def run_head(self, seq, pooled):
        eng = self.eng
        anchor = next(lin for _, lin in eng._head_linears()).weight
        if self.split_head():
            outs = _HeadNode.apply(self, seq, pooled, anchor)
        else:
            outs = _HeadPoolerNode.apply(self, seq, pooled.detach(), anchor)
        return outs


def _alias(t):
    """t as a tensor of its own on the same memory: not an autograd view of the encoder-input buffer, which the other embedding
    kernel writes after t is handed out."""
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage(), t.storage_offset(), t.shape, t.stride())


def _layer_seed(ps, i):
    return ps.st["seed"] + 16 * (i + 1)


def _ly(names, tensors, seed):
    return dict(zip(names, tensors), seed=seed)


class _TextNode(torch.autograd.Function):
    """bert.embeddings: input_ids -> the text rows of the encoder input, (B', Lt, H)."""

    @staticmethod
    def forward(ctx, ps, ids, anchor):
        ps.bind()
        ps.eng._text_fwd(ps.st, ids, ps.x)
        ctx.ps = ps
        ctx.save_for_backward(ids)
        return _alias(ps.view(ps.x)[:, :ps.dims()[1]])

    @staticmethod
    def backward(ctx, dt):
        ps = ctx.ps
        if dt is None or not _engine_runs(ctx.next_functions[1][0], False):
            return None, None, None
        ids, = ctx.saved_tensors
        with ps.eng._node_backward(ps.st, True):
            ps.eng._text_embedding_backward(ps.st, ids, _JoinNode.full(ps, dt, True))
        return None, None, None


class _WordNode(torch.autograd.Function):
    """bert.embeddings.word_embeddings: input_ids -> word[input_ids], fp32 (B', Lt, H), materialised for the hooks. Its backward
    adds the per-token vector gradients into the table rows (cb_embed_word_scatter: one writer and one order per row)."""

    @staticmethod
    def forward(ctx, ps, ids, anchor):
        word = ps.eng._emb("emb.word")[0]
        ctx.ps = ps
        ctx.save_for_backward(ids)
        nseq, lt, _, H = ps.dims()
        return word.index_select(0, ids.reshape(-1).clamp(0, word.shape[0] - 1)).view(nseq, lt, H)

    @staticmethod
    def backward(ctx, dvec):
        ps = ctx.ps
        if dvec is None or not _engine_runs(ctx.next_functions[1][0], False):
            return None, None, None
        ids, = ctx.saved_tensors
        nseq, lt, _, H = ps.dims()
        with ps.eng._node_backward(ps.st, True):
            ops.embed_word_scatter(ids, dvec.reshape(nseq * lt, H).to(torch.float32).contiguous(), ps.eng._emb("emb.word")[1])
        return None, None, None


class _TextVectorsNode(torch.autograd.Function):
    """bert.embeddings with word_embeddings hooked: the word vectors (its output, or a hook's replacement) -> the text rows of the
    encoder input (cb_embed_text_fwd_vectors); the backward returns d vectors (cb_embed_text_bwd_vectors)."""

    @staticmethod
    def forward(ctx, ps, vec, anchor):
        nseq, lt, _, H = ps.dims()
        if tuple(vec.shape) != (nseq, lt, H):
            raise RuntimeError("ClipBertBaseModel: the word vectors handed to bert.embeddings must be (%d, %d, %d), got %s"
                               % (nseq, lt, H, tuple(vec.shape)))
        v = vec.detach().to(torch.float32).reshape(nseq * lt, H)
        if v.stride(1) != 1 or v.stride(0) % 4 or v.data_ptr() % 16:
            v = v.contiguous()
        ps.bind()
        ps.eng._text_vectors_fwd(ps.st, v, ps.x)
        ctx.ps = ps
        ctx.save_for_backward(v)
        return _alias(ps.view(ps.x)[:, :lt])

    @staticmethod
    def backward(ctx, dt):
        ps = ctx.ps
        need_vec, grads = _engine_runs(ctx.next_functions[0][0], True), _engine_runs(ctx.next_functions[1][0], False)
        if dt is None or not (need_vec or grads):
            return None, None, None
        v, = ctx.saved_tensors
        with ps.eng._node_backward(ps.st, grads):
            dvec = ps.eng._text_vectors_backward(ps.st, v, _JoinNode.full(ps, dt, True), grads)
        nseq, lt, _, H = ps.dims()
        return None, dvec.view(nseq, lt, H), None


class _VisualNode(torch.autograd.Function):
    """bert.visual_embeddings: visual_inputs -> the visual rows of the encoder input, (B', Lv, H)."""

    @staticmethod
    def forward(ctx, ps, grid, g, repeat, anchor):
        ps.bind()
        ps.eng._visual_fwd(ps.st, g, repeat, ps.x)
        ctx.ps, ctx.repeat, ctx.grid = ps, repeat, (grid.shape, grid.dtype)
        ctx.save_for_backward(g)
        return _alias(ps.view(ps.x)[:, ps.dims()[1]:])

    @staticmethod
    def backward(ctx, dv):
        ps = ctx.ps
        need_grid, grads = _engine_runs(ctx.next_functions[0][0], True), _engine_runs(ctx.next_functions[2][0], False)
        if dv is None or not (need_grid or grads):
            return None, None, None, None, None
        g, = ctx.saved_tensors
        with ps.eng._node_backward(ps.st, grads):
            dgrid = ps.eng._visual_embedding_backward(ps.st, g, ctx.repeat, _JoinNode.full(ps, dv, False), need_grid, grads)
        if dgrid is not None:
            dgrid = dgrid.view(ctx.grid[0])
        return None, dgrid, None, None, None


class _EmbeddingsNode(torch.autograd.Function):
    """bert.embeddings, bert.visual_embeddings and their concat as one node, for a pass with no hook: visual_inputs -> the encoder
    input (B', L, H). Its backward runs the text, then the visual embedding backward, as the default path does."""

    @staticmethod
    def forward(ctx, ps, grid, anchor):
        st = ps.st
        ps.bind()
        ps.eng._text_fwd(st, st["ids"], ps.x)
        ps.eng._visual_fwd(st, st["grid"], ps.repeat, ps.x)
        ctx.ps, ctx.shape = ps, grid.shape
        return ps.view(ps.x)

    @staticmethod
    def backward(ctx, dx):
        ps = ctx.ps
        need_grid, grads = _engine_runs(ctx.next_functions[0][0], True), _engine_runs(ctx.next_functions[1][0], False)
        if not (need_grid or grads):
            return None, None, None
        with ps.eng._node_backward(ps.st, grads):
            dgrid = ps.eng._embedding_backward(ps.st, ps.dense(dx), need_grid, grads)
        return None, (None if dgrid is None else dgrid.view(ctx.shape)), None


class _JoinNode(torch.autograd.Function):
    """torch.cat([text, visual], 1) (modeling.py:217-220): zero-copy when both are the rows the embeddings wrote."""

    @staticmethod
    def forward(ctx, ps, t, v):
        nseq, lt, L, H = ps.dims()
        ctx.ps = ps
        ot, ov = ps.own.get(id(t)), ps.own.get(id(v))
        if ot is not None and ot[0] is t and ov is not None and ov[0] is v:
            x = ps.x
        else:
            x = torch.empty_like(ps.x)
            xv = x.view(nseq, L, H)
            for part, src, n in ((xv[:, :lt], t, lt), (xv[:, lt:], v, L - lt)):
                if tuple(src.shape) != (nseq, n, H):
                    raise RuntimeError("ClipBertBaseModel: a replaced embedding output must be (%d, %d, %d), got %s"
                                       % (nseq, n, H, tuple(src.shape)))
                part.copy_(src.detach())
        ps.fwd["x_rows"] = x
        return x.view(nseq, L, H)

    @staticmethod
    def backward(ctx, dx):
        ps = ctx.ps
        nseq, lt, L, H = ps.dims()
        g = ps.dense(dx)
        ps.handover["emb"] = g
        gv = g.view(nseq, L, H)
        return None, gv[:, :lt], gv[:, lt:]

    @staticmethod
    def full(ps, g, text):
        """The [B' * L, H] gradient buffer whose text (or visual) rows hold g, for the embedding kernels' row pitch."""
        full = ps.handover.get("emb")
        nseq, lt, L, H = ps.dims()
        if (full is not None and g.dtype == torch.bfloat16 and g.stride() == (L * H, H, 1)
                and g.data_ptr() == full.data_ptr() + (0 if text else lt * H * full.element_size())):
            return full

        buf = torch.zeros(nseq * L, H, dtype=torch.bfloat16, device=g.device)
        v = buf.view(nseq, L, H)
        (v[:, :lt] if text else v[:, lt:]).copy_(g)
        return buf


def _map_outputs(ctx, ps, probs):
    if probs is None:
        probs = torch.empty(0, device=ps.x.device)
    if not ps.diff_attn:
        ctx.mark_non_differentiable(probs)
    return probs


def _dmap(ps, dprobs):
    return None if (dprobs is None or not ps.diff_attn) else dprobs.to(torch.float32).contiguous()


class _LayerModNode(torch.autograd.Function):
    """encoder.layer[i] with none of its sub-modules hooked: hidden_states -> (layer_output, probabilities)."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        eng, st = ps.eng, ps.st
        ps.bind()
        x = ps.rows(h, "the input of encoder.layer[%d]" % i)
        ly, y, probs = eng._layer_fwd(st, i, x, ps.need_backward, ps.want_attn)
        ctx.ps, ctx.i = ps, i
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*(ly[k] for k in _LAYER_STASH))
        ps.fwd["y_rows"] = y
        return ps.view(y), _map_outputs(ctx, ps, probs)

    @staticmethod
    def backward(ctx, dy, dprobs):
        ps, i = ctx.ps, ctx.i
        grads, need_dx = _engine_runs(ctx.next_functions[1][0], False), _engine_runs(ctx.next_functions[0][0], True)
        dattn = _dmap(ps, dprobs)
        if not (grads or need_dx) or (dy is None and dattn is None):
            return None, None, None, None
        ly = _ly(_LAYER_STASH, ctx.saved_tensors, _layer_seed(ps, i))
        dy = torch.zeros_like(ly["x"]) if dy is None else ps.dense(dy)
        with ps.eng._node_backward(ps.st, grads) as sq:
            dxn = ps.eng._layer_backward(ps.st, i, ly, dy, sq, dattn=dattn, grads=grads)
        return None, None, ps.view(dxn), None


class _MapNode(torch.autograd.Function):
    """A_k, encoder.layer[k] split at its differentiable map (layerwise_autograd): hidden_states[k] -> attentions[k]. Its forward
    runs the whole layer and leaves the stash to C_k. Its backward receives the map's full gradient G (the direct term, C_k's
    dO V^T and whatever hooks made of them) and finishes layer k: dQ / dK from G, the QKV weight gradient, the dgrad to
    hidden_states[k]."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        ps.bind()
        x = ps.rows(h, "the input of encoder.layer[%d]" % i)
        ly, y, probs = ps.eng._layer_fwd(ps.st, i, x, ps.need_backward, True)
        ctx.ps, ctx.i = ps, i
        ctx.save_for_backward(x, ly["qkv"], ly["lse"])
        ps.fwd["layer"], ps.fwd["y_rows"] = ly, y
        return probs

    @staticmethod
    def backward(ctx, G):
        ps, i = ctx.ps, ctx.i
        grads = _engine_runs(ctx.next_functions[1][0], False)
        ly = _ly(("x", "qkv", "lse"), ctx.saved_tensors, _layer_seed(ps, i))
        handover = ps.handover.pop(i, None)
        with ps.eng._node_backward(ps.st, grads) as sq:
            dxn = ps.eng._map_backward(ps.st, i, ly, G.to(torch.float32).contiguous(), handover, sq, grads)
        return None, None, ps.view(dxn), None


class _ContextNode(torch.autograd.Function):
    """C_k: (hidden_states[k], attentions[k]) -> hidden_states[k + 1], the reference's dataflow past the map (ctx = A V, output
    projection, LN1, FFN, LN2). Its backward returns d A = dO V^T for the map and nothing for hidden_states[k]: dV and the
    residual ds1 are handed to A_k, which produces the whole gradient at hidden_states[k]."""

    @staticmethod
    def forward(ctx, ps, i, h, a, anchor):
        ly = ps.fwd.pop("layer")
        ctx.ps, ctx.i = ps, i
        ctx.save_for_backward(*(ly[k] for k in _LAYER_STASH))
        return ps.view(ps.fwd["y_rows"])

    @staticmethod
    def backward(ctx, dy):
        ps, i = ctx.ps, ctx.i
        eng, st = ps.eng, ps.st
        nseq, lt, L, H = ps.dims()
        ly = _ly(_LAYER_STASH, ctx.saved_tensors, _layer_seed(ps, i))
        grads = _engine_runs(ctx.next_functions[2][0], False)
        with eng._node_backward(st, grads) as sq:
            wg = eng._wgrad_list()
            du, ds2 = eng._output_backward(st, i, ly, ps.dense(dy), sq, grads, fused=True, wg=wg)
            da = eng._intermediate_backward(st, i, ly, du, sq, grads, ds2, wg=wg)
            dctx, ds1 = eng._self_output_backward(st, i, ly, da, sq, grads, wg=wg)
            eng._issue_wgrads(sq, wg)                       # the QKV weight gradient is A_k's
            dmap = torch.empty(nseq, st["heads"], L, L, dtype=torch.float32, device=dy.device)
            ops.attention_dprobs(ly["qkv"], dctx, dmap, False, nseq, L, st["heads"])
            if _engine_runs(ctx.next_functions[1][0], False):      # A_k runs in this backward: hand dV and ds1 over
                dqkv = torch.empty(nseq * L, 3 * H, dtype=torch.bfloat16, device=dy.device)
                ops.attention_bwd_dv(ly["qkv"], st["mask"], ly["lse"], dctx, dqkv, nseq, L, lt, st["heads"], st["p_a"], ly["seed"] + 1)
                ps.handover[i] = (dqkv, ds1)
        return None, None, None, dmap, None


class _AttentionNode(torch.autograd.Function):
    """layer[i].attention with neither sub-module hooked: hidden_states -> (attention_output (post-LN1), probabilities)."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        eng, st = ps.eng, ps.st
        ps.bind()
        x = ps.rows(h, "the input of layer[%d].attention" % i)
        qkv, c, lse, probs = eng._self_fwd(st, i, x, ps.need_backward, ps.want_attn)
        s1, st1, a = eng._attn_out_fwd(st, i, c, x)
        ctx.ps, ctx.i = ps, i
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, qkv, c, lse, s1, st1)
        ps.fwd["a_rows"] = a
        return ps.view(a), _map_outputs(ctx, ps, probs)

    @staticmethod
    def backward(ctx, da, dprobs):
        ps, i = ctx.ps, ctx.i
        grads, need_dx = _engine_runs(ctx.next_functions[1][0], False), _engine_runs(ctx.next_functions[0][0], True)
        dattn = _dmap(ps, dprobs)
        if not (grads or need_dx) or (da is None and dattn is None):
            return None, None, None, None
        ly = _ly(("x", "qkv", "ctx", "lse", "s1", "st1"), ctx.saved_tensors, _layer_seed(ps, i))
        da = torch.zeros_like(ly["x"]) if da is None else ps.dense(da)
        eng = ps.eng
        with eng._node_backward(ps.st, grads) as sq:
            dctx, ds1 = eng._self_output_backward(ps.st, i, ly, da, sq, grads)
            dxn = eng._self_attention_backward(ps.st, i, ly, dctx, dattn, sq, grads, ds1)
        return None, None, ps.view(dxn), None


class _FfnNode(torch.autograd.Function):
    """layer[i].intermediate + layer[i].output, neither hooked: attention_output -> layer_output (gelu' fused into the dgrad)."""

    @staticmethod
    def forward(ctx, ps, i, a, anchor):
        eng, st = ps.eng, ps.st
        ps.bind()
        ar = ps.rows(a, "the attention output of layer[%d]" % i)
        gel, u = eng._inter_fwd(st, i, ar, ps.need_backward)
        s2, st2, y = eng._out_fwd(st, i, gel, ar)
        ctx.ps, ctx.i = ps, i
        ctx.save_for_backward(ar, u, gel, s2, st2)
        ps.fwd["y_rows"] = y
        return ps.view(y)

    @staticmethod
    def backward(ctx, dy):
        ps, i = ctx.ps, ctx.i
        grads, need_dx = _engine_runs(ctx.next_functions[1][0], False), _engine_runs(ctx.next_functions[0][0], True)
        if not (grads or need_dx):
            return None, None, None, None
        ly = _ly(("a", "u", "gel", "s2", "st2"), ctx.saved_tensors, _layer_seed(ps, i))
        eng = ps.eng
        with eng._node_backward(ps.st, grads) as sq:
            du, ds2 = eng._output_backward(ps.st, i, ly, ps.dense(dy), sq, grads, fused=True)
            da = eng._intermediate_backward(ps.st, i, ly, du, sq, grads, ds2)
        return None, None, ps.view(da), None


class _SelfNode(torch.autograd.Function):
    """layer[i].attention.self: hidden_states -> (context, probabilities). Its backward runs the attention backward with the
    forward's own context (the D = rowsum(dO o O) term belongs to the attention), then the QKV dgrad with the residual gradient
    the attention.output node handed over, if any."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        ps.bind()
        x = ps.rows(h, "the input of layer[%d].attention.self" % i)
        qkv, c, lse, probs = ps.eng._self_fwd(ps.st, i, x, ps.need_backward, ps.want_attn)
        ctx.ps, ctx.i = ps, i
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, qkv, c, lse)
        ps.fwd["ctx_rows"] = c
        return ps.view(c), _map_outputs(ctx, ps, probs)

    @staticmethod
    def backward(ctx, dctx, dprobs):
        ps, i = ctx.ps, ctx.i
        residual = ps.handover.pop(("ds1", i), None)
        grads = _engine_runs(ctx.next_functions[1][0], False)
        dattn = _dmap(ps, dprobs)
        ly = _ly(("x", "qkv", "ctx", "lse"), ctx.saved_tensors, _layer_seed(ps, i))
        if dctx is None and dattn is None:
            return None, None, (None if residual is None else ps.view(residual)), None
        dctx = torch.zeros_like(ly["x"]) if dctx is None else ps.dense(dctx)
        with ps.eng._node_backward(ps.st, grads) as sq:
            dxn = ps.eng._self_attention_backward(ps.st, i, ly, dctx, dattn, sq, grads, residual)
        return None, None, ps.view(dxn), None


class _SelfOutputNode(torch.autograd.Function):
    """layer[i].attention.output: (context, hidden_states) -> attention_output = LN1(dropout(context Wao^T + b) + hidden_states).
    The residual's gradient goes to the self-attention node when that node received the same hidden_states and runs in this
    backward, so that its QKV dgrad adds it in the epilogue (one rounding, as on the default path); else it is returned."""

    @staticmethod
    def forward(ctx, ps, i, c, h, anchor, partner):
        ps.bind()
        cr = ps.rows(c, "the context handed to layer[%d].attention.output" % i)
        x = ps.rows(h, "the hidden states handed to layer[%d].attention.output" % i)
        s1, st1, a = ps.eng._attn_out_fwd(ps.st, i, cr, x)
        ctx.ps, ctx.i, ctx.partner = ps, i, partner
        ctx.save_for_backward(cr, s1, st1)
        ps.fwd["a_rows"] = a
        return ps.view(a)

    @staticmethod
    def backward(ctx, da):
        ps, i = ctx.ps, ctx.i
        grads = _engine_runs(ctx.next_functions[2][0], False)
        ly = _ly(("ctx", "s1", "st1"), ctx.saved_tensors, _layer_seed(ps, i))
        with ps.eng._node_backward(ps.st, grads) as sq:
            dctx, ds1 = ps.eng._self_output_backward(ps.st, i, ly, ps.dense(da), sq, grads)
        if _engine_runs(ctx.partner, False):
            ps.handover[("ds1", i)] = ds1
            return None, None, ps.view(dctx), None, None, None
        return None, None, ps.view(dctx), ps.view(ds1), None, None


class _InterNode(torch.autograd.Function):
    """layer[i].intermediate: attention_output -> GELU output. Its backward multiplies the incoming gradient by the stashed gelu'
    (one bf16 rounding more than the fused dgrad epilogue of the default path), then runs the FFN-up dgrad with the residual
    gradient the output node handed over, if any."""

    @staticmethod
    def forward(ctx, ps, i, a, anchor):
        ps.bind()
        ar = ps.rows(a, "the input of layer[%d].intermediate" % i)
        gel, u = ps.eng._inter_fwd(ps.st, i, ar, ps.need_backward)
        ctx.ps, ctx.i = ps, i
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(ar, u)
        nseq, _, L, _ = ps.dims()
        return gel.view(nseq, L, -1)

    @staticmethod
    def backward(ctx, dgel):
        ps, i = ctx.ps, ctx.i
        residual = ps.handover.pop(("ds2", i), None)
        if dgel is None:
            return None, None, (None if residual is None else ps.view(residual)), None
        grads = _engine_runs(ctx.next_functions[1][0], False)
        ar, u = ctx.saved_tensors
        du = (dgel.reshape(u.shape).float() * u.float()).to(torch.bfloat16)
        with ps.eng._node_backward(ps.st, grads) as sq:
            da = ps.eng._intermediate_backward(ps.st, i, dict(a=ar), du, sq, grads, residual)
        return None, None, ps.view(da), None


class _OutNode(torch.autograd.Function):
    """layer[i].output: (intermediate_output, attention_output) -> layer_output = LN2(dropout(gel Wo^T + b) + attention_output).
    The FFN-down dgrad runs without the gelu' multiply (the hooks see d intermediate_output); the residual's gradient goes to the
    intermediate node under the same rule as _SelfOutputNode's."""

    @staticmethod
    def forward(ctx, ps, i, gel, a, anchor, partner):
        ps.bind()
        nseq, _, L, H = ps.dims()
        n = ps.eng._lin["l%d.inter" % i].n
        if tuple(gel.shape) != (nseq, L, n):
            raise RuntimeError("ClipBertBaseModel: the input of layer[%d].output must be (%d, %d, %d), got %s" % (i, nseq, L, n, tuple(gel.shape)))
        gr = gel.detach().to(torch.bfloat16).reshape(nseq * L, n).contiguous()
        ar = ps.rows(a, "the attention output handed to layer[%d].output" % i)
        s2, st2, y = ps.eng._out_fwd(ps.st, i, gr, ar)
        ctx.ps, ctx.i, ctx.partner = ps, i, partner
        ctx.save_for_backward(gr, s2, st2)
        ps.fwd["y_rows"] = y
        return ps.view(y)

    @staticmethod
    def backward(ctx, dy):
        ps, i = ctx.ps, ctx.i
        grads = _engine_runs(ctx.next_functions[2][0], False)
        ly = _ly(("gel", "s2", "st2"), ctx.saved_tensors, _layer_seed(ps, i))
        with ps.eng._node_backward(ps.st, grads) as sq:
            dgel, ds2 = ps.eng._output_backward(ps.st, i, ly, ps.dense(dy), sq, grads, fused=False)
        nseq, _, L, H = ps.dims()
        dgel = dgel.view(nseq, L, -1)
        if _engine_runs(ctx.partner, False):
            ps.handover[("ds2", i)] = ds2
            return None, None, dgel, None, None, None
        return None, None, dgel, ps.view(ds2), None, None


class _PoolerModNode(torch.autograd.Function):
    """bert.pooler: sequence_output -> pooled_output (tanh' applied on entry to the backward, as one product)."""

    @staticmethod
    def forward(ctx, ps, h, anchor):
        ps.bind()
        x = ps.rows(h, "the input of bert.pooler")
        pooled = ps.eng._pooler_fwd(ps.st, x)
        ctx.ps = ps
        ctx.save_for_backward(x, pooled)
        ps.fwd["seq_rows"] = x
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        ps = ctx.ps
        x, pooled = ctx.saved_tensors
        grads = _engine_runs(ctx.next_functions[1][0], False)
        nseq, _, L, H = ps.dims()
        with ps.eng._node_backward(ps.st, grads):
            dx = ps.eng._pooler_backward(_pooler_pre_grad(pooled, dpooled), x, nseq, L, H, grads)
        return None, ps.view(dx), None


class _HeadNode(torch.autograd.Function):
    """A head's classifier / MLM / ITM part after a hooked pooler: (sequence_output, pooled_output) -> the head's outputs. Its
    backward returns d pooled_output without tanh' (the pooler node applies it: one bf16 rounding more than the default path's
    fused AUX_TANH_GRAD epilogue)."""

    @staticmethod
    def forward(ctx, ps, seq, pooled, anchor):
        return _head_forward(ctx, ps, seq, pooled.detach().to(torch.bfloat16).contiguous())

    @staticmethod
    def backward(ctx, *douts):
        ps = ctx.ps
        grads = _engine_runs(ctx.next_functions[2][0], False)
        nseq, _, L, H = ps.dims()
        st = ctx.st
        with ps.eng._node_backward(st, grads):
            dpooled = ps.eng._head_backward(st, _head_douts(ctx, douts), nseq, H, tanh=False, grads=grads)
            extra = ps.eng._extra_sequence_grad(st)
        return None, (None if extra is None else ps.view(extra)), dpooled, None


class _HeadPoolerNode(torch.autograd.Function):
    """A head's part together with the pooler's backward (pooler not hooked): sequence_output -> the head's outputs, tanh' fused
    into the head's dgrad epilogue as on the default path."""

    @staticmethod
    def forward(ctx, ps, seq, pooled, anchor):
        return _head_forward(ctx, ps, seq, pooled)

    @staticmethod
    def backward(ctx, *douts):
        ps = ctx.ps
        grads = _engine_runs(ctx.next_functions[2][0], False)
        nseq, _, L, H = ps.dims()
        st = ctx.st
        with ps.eng._node_backward(st, grads):
            dpre = ps.eng._head_backward(st, _head_douts(ctx, douts), nseq, H, grads=grads)
            dx = ps.eng._pooler_backward(dpre, st["x_last"], nseq, L, H, grads)
            extra = ps.eng._extra_sequence_grad(st)
            if extra is not None:
                dx += extra
        return None, ps.view(dx), None, None


def _head_forward(ctx, ps, seq, pooled):
    eng = ps.eng
    ps.bind()
    x = ps.fwd.pop("seq_rows", None)
    if x is None or ps.fwd.get("seq") is not seq:
        x = ps.rows(seq, "the sequence output handed to the head")
    st = dict(ps.st, x_last=x, pooled=pooled)
    nseq = ps.dims()[0]
    outs = eng._head_forward(pooled, st, nseq, st["p_h"], st["seed"], ps.need_backward)
    ctx.ps, ctx.st = ps, st
    ctx.set_materialize_grads(False)
    ctx.multi = isinstance(outs, tuple)
    return outs


def _head_douts(ctx, douts):
    return douts if ctx.multi else douts[0]


class _ClipBertHeadModel(nn.Module):
    """Shared engine: ClipBertBaseModel + an MLP head; subclasses set the head and the loss."""

    def __init__(self, config, bert=None):
        super().__init__()
        self.config = config
        self.bert = ClipBertBaseModel(config, _engine=self) if bert is None else bert
        self.dropout = nn.Dropout(_cfg(config, "hidden_dropout_prob"))
        self._flat = None
        self._dirty = True
        self._call_count = 0
        self._seed_base = None
        self._drop_counter = None   # uint64 device word: the dropout stream position, advanced ON THE DEVICE once per training forward
        self._capture = None     # tests set this to a dict to receive per-layer activations (and, in backward, gradients)
        self._inject = None      # tests: {layer index: (B', L, 768) hidden state} makes that encoder layer start from the given tensor
        self._pending_backward = 0
        self._grad_ready_hook = None
        self._optimizer_emits_packed = False   # FusedAdamW writes the bf16 operands itself (clipbert_b200/optim.py)

    # ---- flat parameter storage -------------------------------------------------------------------
    def _head_linears(self):
        raise NotImplementedError

    def _ensure_ready(self, device):
        if self._flat is None or not self._flat.is_current() or self._flat.device != device:
            self._build_flat(device)
            self._dirty = True
        if self._dirty or self._flat.needs_repack():
            self._repack()
            self._dirty = False
            self._flat.needs_repack()

    def mark_weights_updated(self):
        self._dirty = True

    # ---- FusedAdamW hooks (clipbert_b200/optim.py) -------------------------------------------------
    def optimizer_segments(self):
        """Linear weights (the prefix of the flat buffer) have a bf16 tensor-core copy; biases, LayerNorm and embedding
        tables are consumed in fp32."""
        f = self._flat
        return [dict(param=e["param"], row_len=0, scale_off=-1, emit=e["offset"] + e["numel"] <= f.packed_prefix) for e in f.entries]

    def optimizer_scales(self):
        return None

    def packed_written_by_optimizer(self):
        self._dirty = False
        self._flat.needs_repack()

    def _add_linear(self, flat, name, lins, pad_rows=None):
        """Register weight(s) then bias(es) of one or several nn.Linear (fused along the output dim)."""
        ews = [flat.add(name + ".w%d" % i, l.weight) for i, l in enumerate(lins[:-1])]
        n = sum(l.weight.shape[0] for l in lins)
        k = lins[0].weight.shape[1]
        npad = n if pad_rows is None else pad_rows
        last_rows = lins[-1].weight.shape[0] + (npad - n)
        ews.append(flat.add(name + ".w%d" % (len(lins) - 1), lins[-1].weight, slot_numel=last_rows * k))
        ebs = [flat.add(name + ".b%d" % i, l.bias) for i, l in enumerate(lins[:-1])]
        ebs.append(flat.add(name + ".b%d" % (len(lins) - 1), lins[-1].bias, slot_numel=lins[-1].bias.shape[0] + (npad - n)))
        # fused layout requires contiguity of the pieces: every piece but the last must fill its slot
        for e in ews[:-1] + ebs[:-1]:
            assert e["numel"] == e["slot"], "fused linear pieces must be multiples of %d elements" % 64
        return dict(w_off=ews[0]["offset"], b_off=ebs[0]["offset"], n=npad, k=k)

    def _build_flat(self, device):
        flat = FlatGroup(device)
        self._spec = {}
        bert = self.bert
        for i, layer in enumerate(bert.encoder.layer):
            att = layer.attention
            self._spec["l%d.qkv" % i] = self._add_linear(flat, "l%d.qkv" % i, [att.self.query, att.self.key, att.self.value])
            self._spec["l%d.ao" % i] = self._add_linear(flat, "l%d.ao" % i, [att.output.dense])
            self._spec["l%d.ln1" % i] = (flat.add("l%d.ln1.w" % i, att.output.LayerNorm.weight), flat.add("l%d.ln1.b" % i, att.output.LayerNorm.bias))
            self._spec["l%d.inter" % i] = self._add_linear(flat, "l%d.inter" % i, [layer.intermediate.dense])
            self._spec["l%d.out" % i] = self._add_linear(flat, "l%d.out" % i, [layer.output.dense])
            self._spec["l%d.ln2" % i] = (flat.add("l%d.ln2.w" % i, layer.output.LayerNorm.weight), flat.add("l%d.ln2.b" % i, layer.output.LayerNorm.bias))
        self._spec["pooler"] = self._add_linear(flat, "pooler", [bert.pooler.dense])
        for name, lin in self._head_linears():
            n = lin.weight.shape[0]
            self._spec[name] = self._add_linear(flat, name, [lin], pad_rows=(n + 7) // 8 * 8)
        for name, ln in self._extra_layernorms():
            self._spec[name] = (flat.add(name + ".w", ln.weight), flat.add(name + ".b", ln.bias))
        flat.mark_packed_prefix()
        emb, vis = bert.embeddings, bert.visual_embeddings
        self._spec["emb.ln"] = (flat.add("emb.ln.w", emb.LayerNorm.weight), flat.add("emb.ln.b", emb.LayerNorm.bias))
        self._spec["vis.ln"] = (flat.add("vis.ln.w", vis.LayerNorm.weight), flat.add("vis.ln.b", vis.LayerNorm.bias))
        # the word table gets room for 8-row padding: the tied MLM decoder reads / accumulates it as a [vocab_pad, 768] operand
        vocab_pad = (emb.word_embeddings.weight.shape[0] + 7) // 8 * 8
        self._spec["emb.word"] = flat.add("emb.word", emb.word_embeddings.weight, slot_numel=vocab_pad * emb.word_embeddings.weight.shape[1])
        for key, mod in (("emb.pos", emb.position_embeddings), ("emb.type", emb.token_type_embeddings),
                         ("vis.pos", vis.position_embeddings), ("vis.row", vis.row_position_embeddings),
                         ("vis.col", vis.col_position_embeddings), ("vis.type", vis.token_type_embeddings)):
            self._spec[key] = flat.add(key, mod.weight)
        for name, p, slot in self._extra_params():
            self._spec[name] = flat.add(name, p, slot_numel=slot)
        flat.materialize()
        self._flat = flat
        # resolve views
        self._lin = {}
        for key, sp in self._spec.items():
            if isinstance(sp, dict) and "w_off" in sp:
                li = _Lin()
                n, k = sp["n"], sp["k"]
                li.n, li.k = n, k
                li.w = flat.packed[sp["w_off"]: sp["w_off"] + n * k].view(n, k)
                li.gw = flat.grad[sp["w_off"]: sp["w_off"] + n * k].view(n, k)
                li.b = flat.master[sp["b_off"]: sp["b_off"] + n]
                li.gb = flat.grad[sp["b_off"]: sp["b_off"] + n]
                self._lin[key] = li

    def _extra_layernorms(self):
        return []

    def _extra_params(self):
        return []

    def _ln(self, key):
        ew, eb = self._spec[key]
        f = self._flat
        return (f.master[ew["offset"]: ew["offset"] + ew["numel"]], f.master[eb["offset"]: eb["offset"] + eb["numel"]],
                f.grad[ew["offset"]: ew["offset"] + ew["numel"]], f.grad[eb["offset"]: eb["offset"] + eb["numel"]])

    def _emb(self, key):
        e = self._spec[key]
        f = self._flat
        shape = e["param"].shape
        return (f.master[e["offset"]: e["offset"] + e["numel"]].view(shape), f.grad[e["offset"]: e["offset"] + e["numel"]].view(shape))

    @torch.no_grad()
    def _repack(self):
        """fp32 masters -> bf16 tensor-core operands: ONE cast kernel over the linear-weight prefix."""
        f = self._flat
        n = f.packed_prefix
        ops.cast_scale(f.master[:n], f.packed[:n])

    # ---- seeds ------------------------------------------------------------------------------------
    def _next_seed(self):
        if self._seed_base is None:
            self._seed_base = torch.initial_seed() & 0xFFFFFFFFFFFF
        self._call_count += 1
        return (self._seed_base + self._call_count * 1000003) & 0xFFFFFFFFFFFFFFFF

    def _advance_dropout_stream(self, dev):
        """The reference draws fresh masks at every call (nn.Dropout, transformers.py:170,222,295,375). The seed above is a
        host value - a captured CUDA graph would bake it in and replay the same masks - so the stream position also lives in
        device memory: one tiny kernel increments the model's counter and writes the new value to a per-call word; every
        mask-drawing launch of this forward AND of its backward reads that word when it runs (ops.dropout_offset_bind).
        Returns the per-call word."""
        if self._drop_counter is None or self._drop_counter.device != dev:
            self._drop_counter = torch.zeros(1, dtype=torch.int64, device=dev)
        word = torch.empty(1, dtype=torch.int64, device=dev)
        ops.dropout_offset_advance(self._drop_counter, word)
        return word

    # ---- forward ----------------------------------------------------------------------------------
    def _run(self, text_input_ids, visual_inputs, text_input_mask, repeat_counts=None):
        """Returns fp32 logits (B', num_outputs). visual_inputs: (B or B', T, h, w, 768)."""
        _require_cuda(text_input_ids)
        dev = text_input_ids.device
        self._ensure_ready(dev)
        nseq = text_input_ids.shape[0]
        nvid = visual_inputs.shape[0]
        if repeat_counts is None:
            assert nvid == nseq, "visual_inputs must have one row per text example (or pass repeat counts)"
            repeat = (1, None, None)
        else:
            assert len(repeat_counts) == nvid and sum(repeat_counts) == nseq
            if sum(repeat_counts) == len(repeat_counts):
                # repeat_tensor_rows returns its input untouched in this case, even for counts like [2, 0, 1]
                # (src/datasets/data_utils.py:351) - follow the reference
                repeat = (1, None, None)
            elif len(set(repeat_counts)) == 1:
                repeat = (int(repeat_counts[0]), None, None)
            else:
                s2v = torch.tensor([i for i, r in enumerate(repeat_counts) for _ in range(r)], dtype=torch.int32)
                starts = torch.tensor([0] + list(torch.tensor(repeat_counts).cumsum(0)), dtype=torch.int32)
                repeat = (0, s2v.to(dev), starts.to(dev))
        hooked = self._bert_hooked()
        if hooked:
            return self._run_modules(text_input_ids, visual_inputs, text_input_mask, repeat, hooked)
        grid = visual_inputs
        if grid.dtype != torch.bfloat16:
            grid = grid.to(torch.bfloat16)
        grid = grid.contiguous()
        ids = text_input_ids.contiguous()
        mask = text_input_mask.to(torch.int64).contiguous()
        if torch.is_grad_enabled() and (grid.requires_grad or any(p.requires_grad for p in self.parameters())):
            # a grid that requires grad keeps a fully frozen head on the graph (gradients to the frames), as in _run_base
            anchor = self.bert.pooler.dense.weight
            return _TransformerFn.apply(self, grid, anchor, ids, mask, repeat)
        return self._forward_impl(ids, grid, mask, repeat, need_backward=False)[0]

    def _run_base(self, text_input_ids, visual_inputs, attention_mask, want_hidden, want_attn, diff_attn, records):
        """ClipBertBaseModel.forward on this engine's default path (the head itself is not run), one autograd node when the pass
        records autograd (_base_pass). visual_inputs: (B', T, h, w, 768)."""
        _require_cuda(text_input_ids)
        self._ensure_ready(text_input_ids.device)
        assert visual_inputs.shape[0] == text_input_ids.shape[0], "visual_inputs must have one row per text example"
        grid = visual_inputs if visual_inputs.dtype == torch.bfloat16 else visual_inputs.to(torch.bfloat16)
        grid = grid.contiguous()
        ids = text_input_ids.contiguous()
        mask = attention_mask.to(torch.int64).contiguous()
        flags = (bool(want_hidden), bool(want_attn), bool(want_attn and diff_attn))
        if records:
            outs = _BaseModelFn.apply(self, grid, self.bert.pooler.dense.weight, ids, mask, flags)
            n_hidden = len(self.bert.encoder.layer) + 1 if flags[0] else 0
            seq, pooled, hidden, attn = outs[0], outs[1], outs[2:2 + n_hidden], outs[2 + n_hidden:]
        else:
            seq, pooled, hidden, attn = self._forward_impl(ids, grid, mask, (1, None, None), need_backward=False, base=flags)[0]
        out = (seq, pooled)
        if flags[0]:
            out = out + (tuple(hidden),)
        if flags[1]:
            out = out + (tuple(attn),)
        return out

    def _base_pass(self, visual_inputs):
        """Which path a bert(...) call takes: (the module-path pass to run it in, or None for the default path; whether the pass
        records autograd). The module path serves a hook on bert or a module below it, and layerwise_autograd on a pass that
        records autograd (the maps split when differentiable_attentions is on). Raises for the combinations that are refused."""
        hooked = self._bert_hooked()
        if hooked:
            return _BertPass(self, hooked), None
        bert = self.bert
        records = torch.is_grad_enabled() and (visual_inputs.requires_grad or any(p.requires_grad for p in bert.parameters()))
        if not records:
            return None, False
        if bert.recompute_activations and (bert.differentiable_attentions or bert.layerwise_autograd):
            raise RuntimeError("ClipBertBaseModel: recompute_activations cannot be combined with %s: its backward reads every "
                               "layer's activations; turn one of the switches off" %
                               ("differentiable_attentions" if bert.differentiable_attentions else "layerwise_autograd"))
        if not bert.layerwise_autograd:
            return None, True
        if self._grad_ready_hook is not None:
            raise RuntimeError("ClipBertBaseModel.layerwise_autograd is for analysis, not data-parallel training: it cannot run while "
                               "the overlapped gradient exchange (enable_overlapped_allreduce) is enabled")
        return _BertPass(self, set(), split_maps=bert.output_attentions and bert.differentiable_attentions), True

    # ---- module path: hooks on bert and the modules below it ---------------------------------------------------------------
    def _bert_sites(self):
        """([(name, module, the name of the module to hook instead or None when the module itself is hookable, whether it is one
        of the head's own modules)], {module: its encoder layer}, the sites' hook dicts), computed once."""
        sites = self.__dict__.get("_bert_site_cache")
        if sites is None:
            bert = self.bert
            by_name = dict(bert.named_modules(prefix="bert"))
            sites = []
            for name, mod in by_name.items():
                instead = None
                if not isinstance(mod, _BERT_SITES):
                    instead = name
                    while not isinstance(by_name.get(instead), _BERT_SITES):
                        instead = instead.rsplit(".", 1)[0]
                sites.append((name, mod, instead, False))
            inside = set(by_name.values())
            sites += [(name, mod, None, True) for name, mod in self.named_modules() if mod is not self and mod not in inside]
            index = {m: i for i, layer in enumerate(bert.encoder.layer) for m in layer.modules()}
            # the hook registries of every site (torch adds hooks to these dicts in place): the no-hook check in one C loop
            dicts = tuple(d for _, m, _, _ in sites for d in (m._forward_hooks, m._forward_pre_hooks, m._backward_hooks,
                                                              m._backward_pre_hooks))
            self.__dict__["_bert_site_cache"] = sites = (sites, index, dicts)
        return sites

    def _bert_site_index(self):
        return self._bert_sites()[1]

    def _bert_hooked(self):
        """The set of bert's modules the forward must call because a hook is registered on them (all of them when a global module
        hook exists); empty: the default path. Raises for hooks that cannot be honoured."""
        glob = _global_hooks()
        sites, _, hook_dicts = self._bert_sites()
        if not glob and not any(map(len, hook_dicts)):
            return set()
        hooked = set()
        for name, mod, instead, in_head in sites:
            if not _has_hooks(mod):
                if glob and instead is None and not in_head:
                    hooked.add(mod)
                continue
            if in_head:
                raise RuntimeError("%s: hooks on the head's own module %s are not supported: the head's layers run fused behind its "
                                   "forward; hook the head itself or a module of its bert" % (type(self).__name__, name))
            if instead is not None:
                raise RuntimeError("ClipBertBaseModel: hooks on %s are not supported: it runs fused into a kernel of its parent and its "
                                   "output never exists in memory; hook %s instead" % (name, instead))
            hooked.add(mod)
        if hooked and self._grad_ready_hook is not None:
            raise RuntimeError("ClipBertBaseModel: hooks on the transformer's modules are for analysis, not data-parallel training: "
                               "they cannot run while the overlapped gradient exchange (enable_overlapped_allreduce) is enabled")
        if hooked and self.bert.recompute_activations and torch.is_grad_enabled():
            raise RuntimeError("ClipBertBaseModel: recompute_activations cannot be combined with hooks on the transformer's modules: "
                               "the module path keeps every layer's activations for its nodes' backward; remove the hooks or turn "
                               "the switch off")
        return hooked

    def _run_modules(self, ids, visual_inputs, mask, repeat, hooked):
        """The head's forward with bert on the module path: bert(...) called as a module (torch's hooks on it and below it fire),
        then the head's part as one node. With repeat counts, the (B', T, h, w, 768) rows of repeat_tensor_rows are materialised
        for the hooks only when a hook on bert or bert.visual_embeddings can see them, and then as a detached copy: unless a hook
        replaces them, the visual-embedding kernel still repeats the head's grid and sums its gradient, as on the default path."""
        bert = self.bert
        given = visual_inputs
        if repeat[0] != 1 and (bert in hooked or bert.visual_embeddings in hooked):
            g = visual_inputs.detach()
            given = g.repeat_interleave(repeat[0], 0) if repeat[0] > 1 else g.index_select(0, repeat[1].to(torch.int64))
        with _BertPass(self, hooked, repeat, (given, visual_inputs)) as ps:
            out = bert(ids, given, mask)
            return ps.run_head(out[0], out[1])

    @contextlib.contextmanager
    def _node_backward(self, st, grads):
        """Around the backward of one module-path node: the pass's dropout word bound (its masks regenerated) and unbound on the way
        out, the node's side-queue weight gradients joined before it returns (a partial backward may run no later node), and,
        when it writes parameter gradients, the flat buffer attached and the bf16 operands due a repack."""
        ops.dropout_offset_bind(st["drop_word"])
        sq = ops.SideQueue()
        try:
            if grads:
                self._flat.attach_grads()
            yield sq
            if grads and not self._optimizer_emits_packed:
                self._dirty = True
        finally:
            sq.join()
            ops.dropout_offset_bind(None)

    def _backward_done(self):
        self._pending_backward = max(0, self._pending_backward - 1)
        if self._pending_backward == 0 and self._grad_ready_hook is not None:
            self._grad_ready_hook(self._flat.grad)          # every clip's contribution is in: the exchange may start

    def _gemm_fwd(self, x, m, li, out, **kw):
        ops.gemm(mode=ops.CB_GEMM_TN, m=m, n=li.n, k=li.k, a=x, a_rows=m, a_ld=kw.pop("a_ld", li.k), b=li.w, b_rows=li.n, b_ld=li.k,
                 shift=li.b, out=out, out_ld=li.n, **kw)

    def _forward_impl(self, ids, grid, mask, repeat, need_backward, base=None):
        """Binds the per-call dropout word for the duration of the pass and unbinds it on the way out: the binding is process-wide
        state of the library, and a word that outlives its tensor would be a dangling device pointer for every later launch that
        draws masks (found by the autotuner: cb_gemm launches with dropout after the recording step's tensors had been freed)."""
        try:
            return self._forward_body(ids, grid, mask, repeat, need_backward, base)
        finally:
            ops.dropout_offset_bind(None)

    def _forward_body(self, ids, grid, mask, repeat, need_backward, base=None):
        """base = None: the head's forward, returns its outputs. base = (want_hidden, want_attn): ClipBertBaseModel.forward,
        returns (sequence_output, pooled_output, hidden_states, attentions) without running the head."""
        want_hidden, want_attn = base[:2] if base is not None else (False, False)
        st = self._pass_state(ids, grid, mask, repeat, self.bert.training if base is not None else self.training)
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        H, M, seed, p_h = st["H"], nseq * L, st["seed"], st["p_h"]
        # ---- embeddings: [text ; visual] written straight into one (B', L, 768) buffer ----
        x = torch.empty(M, H, dtype=torch.bfloat16, device=ids.device)
        self._text_fwd(st, ids, x)
        self._visual_fwd(st, st["grid"], repeat, x)
        cap = self._capture
        if cap is not None:
            cap["embeddings"] = x.view(nseq, L, H).clone()
            cap.update(seed=seed, drop_word=st["drop_word"], stats_t=st["stats_t"], stats_v=st["stats_v"], grid=st["grid"],
                       idx=None if st["sample"] is None else st["sample"][0], row_tab=st["row_tab"], col_tab=st["col_tab"])
        # ---- encoder ----
        hidden, attn = [], []
        recompute = need_backward and self.bert.recompute_activations
        for i in range(len(self.bert.encoder.layer)):
            if self._inject is not None and i in self._inject:      # test hook: layer-local parity (same input on both sides)
                x = self._inject[i].to(device=ids.device, dtype=torch.bfloat16).reshape(M, H).contiguous()
            if want_hidden:
                hidden.append(x.view(nseq, L, H))
            ly, y, probs = self._layer_fwd(st, i, x, need_backward, want_attn)
            if want_attn:
                attn.append(probs)
            ls = seed + 16 * (i + 1)
            if need_backward and recompute:
                st["layers"].append(dict(x=x, seed=ls, recompute=True))    # the rest is re-run before the layer's backward
            elif need_backward:
                st["layers"].append(dict(ly, seed=ls))
            if cap is not None:
                cap["l%d" % i] = ly
            x = y
            if cap is not None:
                cap["layer%d" % i] = x.view(nseq, L, H)
        st["x_last"] = x
        pooled = self._pooler_fwd(st, x)
        st["pooled"] = pooled
        if cap is not None:
            cap["pooled"] = pooled
        if base is not None:
            if want_hidden:
                hidden.append(x.view(nseq, L, H))
            out = (x.view(nseq, L, H), pooled, hidden, attn)
        else:
            out = self._head_forward(pooled, st, nseq, p_h, seed, need_backward)
        return out, (st if need_backward else None)

    # ---- the forward's per-module pieces: the default path calls them in this order, the module path from the modules ------
    def _pass_state(self, ids, grid, mask, repeat, train):
        """The state one forward pass shares: its seed, dropout probabilities and word (drawn and bound here), dims, the visual
        grid and position tables (a sampled subset in pre-training), the embedding stats, and the per-layer stash list."""
        dev = ids.device
        cfg = self.config
        H = _cfg(cfg, "hidden_size")
        p_h = float(_cfg(cfg, "hidden_dropout_prob")) if train else 0.0
        p_a = float(_cfg(cfg, "attention_probs_dropout_prob")) if train else 0.0
        seed = self._next_seed()
        nseq, lt = ids.shape
        nvid, T, gh, gw, _ = grid.shape
        f32 = torch.float32
        # ---- pre-training only, train mode only: keep a random subset of the visual tokens (modeling.py:80-88) ----
        # The kept positions are the same for every sequence of the batch, so the subset is presented to the embedding kernels
        # as a (n_keep x 1) grid whose "row" table is row[idx // w] + col[idx % w] (its "column" table is one zero row): index
        # bookkeeping on the host, arithmetic in the same kernels. (The host draw makes such a step not graph-capturable.)
        row_tab, col_tab = self._emb("vis.row")[0], self._emb("vis.col")[0]
        sample = None
        n_keep = int(_cfg(cfg, "pixel_random_sampling_size", 0) or 0)
        if n_keep > 0 and train and n_keep < gh * gw:
            idx = get_random_sample_indices(gh * gw, n_keep, dev)
            grid = grid.view(nvid, T, gh * gw, H).index_select(2, idx).view(nvid, T, n_keep, 1, H)
            row_tab = (row_tab[idx // gw] + col_tab[idx % gw]).contiguous()
            col_tab = torch.zeros(1, H, dtype=f32, device=dev)
            sample = (idx, gh, gw, row_tab, col_tab)
            gh, gw = n_keep, 1
        drop_word = self._advance_dropout_stream(dev) if (p_h > 0 or p_a > 0) else None
        ops.dropout_offset_bind(drop_word)
        return dict(ids=ids, mask=mask, grid=grid, repeat=repeat, seed=seed, p_h=p_h, p_a=p_a, dims=(nseq, nvid, T, gh, gw, lt, lt + gh * gw),
                    layers=[], sample=sample, drop_word=drop_word, row_tab=row_tab, col_tab=col_tab, H=H,
                    heads=_cfg(cfg, "num_attention_heads"), eps=float(_cfg(cfg, "layer_norm_eps")),
                    stats_t=torch.empty(nseq * lt, 2, dtype=f32, device=dev), stats_v=torch.empty(nseq * gh * gw, 2, dtype=f32, device=dev))

    def _text_fwd(self, st, ids, x):
        """BertEmbeddings: LN(word[ids] + pos + type[0]) and dropout into the text rows of x ([B' * L, H], row pitch L * H)."""
        nseq, _, _, _, _, lt, L = st["dims"]
        g_t, b_t, _, _ = self._ln("emb.ln")
        word, pos, typ = self._emb("emb.word")[0], self._emb("emb.pos")[0], self._emb("emb.type")[0]
        ops.embed_text_fwd(ids, word, pos, typ, g_t, b_t, x, st["stats_t"], nseq, lt, L, st["eps"], st["p_h"], st["seed"] + 1)

    def _text_vectors_fwd(self, st, vec, x):
        """BertEmbeddings from fp32 word vectors vec ([B' * Lt, H] rows, any row pitch): LN(vec + pos + type[0]) and dropout."""
        nseq, _, _, _, _, lt, L = st["dims"]
        g_t, b_t, _, _ = self._ln("emb.ln")
        ops.embed_text_fwd_vectors(vec, self._emb("emb.pos")[0], self._emb("emb.type")[0], g_t, b_t, x, st["stats_t"], nseq, lt, L,
                                   st["eps"], st["p_h"], st["seed"] + 1)

    def _visual_fwd(self, st, grid, repeat, x):
        """VisualInputEmbedding: frame mean, + row / col / type, LN and dropout into the visual rows of x."""
        nseq, _, T, gh, gw, lt, L = st["dims"]
        n_ex, s2v, _ = repeat
        g_v, b_v, _, _ = self._ln("vis.ln")
        ops.embed_visual_fwd(grid, s2v, n_ex, st["row_tab"], st["col_tab"], self._emb("vis.type")[0], g_v, b_v,
                             x, st["stats_v"], nseq, T, gh, gw, lt, L, st["eps"], st["p_h"], st["seed"] + 2)

    def _self_fwd(self, st, i, x, need_backward, want_attn):
        """BertSelfAttention of layer i from its input rows x: (qkv, context, lse or None, post-dropout probabilities or None)."""
        nseq, _, _, _, _, lt, L = st["dims"]
        H, heads, M, dev = st["H"], st["heads"], nseq * L, x.device
        ls = st["seed"] + 16 * (i + 1)
        qkv = torch.empty(M, 3 * H, dtype=torch.bfloat16, device=dev)
        self._gemm_fwd(x, M, self._lin["l%d.qkv" % i], qkv)
        ctx = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(nseq, heads, L, dtype=torch.float32, device=dev) if (need_backward or want_attn) else None
        ops.attention_fwd(qkv, st["mask"], ctx, lse, nseq, L, lt, heads, st["p_a"], ls + 1)
        probs = None
        if want_attn:       # same seed and bound word as the forward: the probabilities its context was made from
            probs = torch.empty(nseq, heads, L, L, dtype=torch.float32, device=dev)
            ops.attention_probs(qkv, st["mask"], lse, probs, nseq, L, lt, heads, st["p_a"], ls + 1)
        if self._capture is not None:      # test hook: what layer i's maps are made from, on the default and the module path
            self._capture["attn%d" % i] = dict(qkv=qkv, lse=lse, seed=ls + 1, word=st["drop_word"])
        return qkv, ctx, lse, probs

    def _attn_out_fwd(self, st, i, ctx, x):
        """BertSelfOutput: a = LN1(dropout(ctx Wao^T + b) + x); returns (s1, its LN stats, a)."""
        M, H, dev = ctx.shape[0], st["H"], ctx.device
        g1, b1, _, _ = self._ln("l%d.ln1" % i)
        s1 = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        self._gemm_fwd(ctx, M, self._lin["l%d.ao" % i], s1, residual=x, res_ld=H, dropout_p=st["p_h"], dropout_seed=st["seed"] + 16 * (i + 1) + 2)
        a = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        st1 = torch.empty(M, 2, dtype=torch.float32, device=dev)
        ops.layernorm_fwd(s1, g1, b1, a, st1, st["eps"])
        return s1, st1, a

    def _inter_fwd(self, st, i, a, need_backward):
        """BertIntermediate: (gel = GELU(a Win^T + b), u = gelu'(pre-activation) or None)."""
        M, dev = a.shape[0], a.device
        in_l = self._lin["l%d.inter" % i]
        gel = torch.empty(M, in_l.n, dtype=torch.bfloat16, device=dev)
        u = None
        if need_backward:
            # u holds gelu'(pre-activation), not the pre-activation: the backward epilogue is then one multiply
            u = torch.empty(M, in_l.n, dtype=torch.bfloat16, device=dev)
            self._gemm_fwd(a, M, in_l, gel, act=ops.ACT_GELU_STASH_GRAD, out2=u, out2_ld=in_l.n)
        else:
            self._gemm_fwd(a, M, in_l, gel, act=ops.ACT_GELU)
        return gel, u

    def _out_fwd(self, st, i, gel, a):
        """BertOutput: y = LN2(dropout(gel Wo^T + b) + a); returns (s2, its LN stats, y)."""
        M, H, dev = gel.shape[0], st["H"], gel.device
        g2, b2, _, _ = self._ln("l%d.ln2" % i)
        s2 = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        self._gemm_fwd(gel, M, self._lin["l%d.out" % i], s2, residual=a, res_ld=H, dropout_p=st["p_h"], dropout_seed=st["seed"] + 16 * (i + 1) + 3)
        y = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        st2 = torch.empty(M, 2, dtype=torch.float32, device=dev)
        ops.layernorm_fwd(s2, g2, b2, y, st2, st["eps"])
        return s2, st2, y

    def _layer_fwd(self, st, i, x, need_backward, want_attn):
        """BertLayer i from its input rows x: (its stash {x, qkv, ctx, lse, s1, st1, a, u, gel, s2, st2}, the output rows, the
        post-dropout probabilities or None)."""
        qkv, ctx, lse, probs = self._self_fwd(st, i, x, need_backward, want_attn)
        s1, st1, a = self._attn_out_fwd(st, i, ctx, x)
        gel, u = self._inter_fwd(st, i, a, need_backward)
        s2, st2, y = self._out_fwd(st, i, gel, a)
        return dict(x=x, qkv=qkv, ctx=ctx, lse=lse, s1=s1, st1=st1, a=a, u=u, gel=gel, s2=s2, st2=st2), y, probs

    def _pooler_fwd(self, st, x):
        """BertPooler on the [CLS] rows of x (row pitch L * H, no gather)."""
        nseq, L = st["dims"][0], st["dims"][6]
        pooled = torch.empty(nseq, st["H"], dtype=torch.bfloat16, device=x.device)
        self._gemm_fwd(x, nseq, self._lin["pooler"], pooled, a_ld=L * st["H"], act=ops.ACT_TANH)
        return pooled

    # generic 2-layer MLP head: dropout -> Linear -> ReLU -> Linear (modeling.py:534-539,552-553)
    def _mlp_head_forward(self, pooled, st, nseq, p_h, seed, num_out):
        dev = pooled.device
        c0, c2 = self._lin["cls0"], self._lin["cls2"]
        if p_h > 0:
            pd = torch.empty_like(pooled)
            ops.dropout(pooled, pd, p_h, seed + 5)
        else:
            pd = pooled
        c1 = torch.empty(nseq, c0.n, dtype=torch.bfloat16, device=dev)
        self._gemm_fwd(pd, nseq, c0, c1, act=ops.ACT_RELU)
        logits = torch.empty(nseq, c2.n, dtype=torch.float32, device=dev)
        self._gemm_fwd(c1, nseq, c2, logits, out_fp32=1)
        st["pd"], st["c1"], st["num_out"] = pd, c1, num_out
        if self._capture is not None:
            self._capture.update(pd=pd, c1=c1, logits=logits)
        return logits[:, :num_out]

    def _head_forward(self, pooled, st, nseq, p_h, seed, need_backward):
        return self._mlp_head_forward(pooled, st, nseq, p_h, seed, self._num_head_outputs())

    # ---- backward ---------------------------------------------------------------------------------
    def _wgrad_kw(self, li, dy, x, rows, x_ld=None):
        return dict(mode=ops.CB_GEMM_WGRAD, m=li.n, n=li.k, k=rows, a=dy, a_rows=rows, a_ld=li.n, b=x, b_rows=rows,
                    b_ld=li.k if x_ld is None else x_ld, out=li.gw, out_ld=li.k, out_fp32=1)

    def _wgrad(self, li, dy, x, rows, x_ld=None):
        ops.gemm(**self._wgrad_kw(li, dy, x, rows, x_ld))

    def _split_wgrad_kw(self, key, li, dy, x, rows):
        """A weight gradient of an encoder layer launched on its own: one launch, pinned to the tile width and K-split of the
        grouped launch _layer_backward issues for it (ops.group_wgrad: the layer's four, or its FFN and attention pairs), so that
        each element is summed in the same order and observe-only hooks keep the bits."""
        kw = self._wgrad_kw(li, dy, x, rows)
        gmode = ops.group_wgrad
        if gmode not in (1, 3, 4) or not dy.is_cuda:
            return kw
        cache = self.__dict__.setdefault("_wgrad_pins", {})
        pins = cache.get((rows, gmode))
        if pins is None:
            lins = {k: self._lin["l0.%s" % k] for k in ("out", "inter", "ao", "qkv")}
            pins = {}
            for grp in ([("out", "inter"), ("ao", "qkv")] if gmode == 4 else [("out", "inter", "ao", "qkv")]):
                # the plan query reads the descriptors' shapes only
                plan = ops.gemm_wgrad_group_plan([self._wgrad_kw(lins[k], lins[k].gw, lins[k].gw, rows) for k in grp])
                pins.update({k: plan for k in grp})
            cache[(rows, gmode)] = pins
        if pins[key] is None:
            return kw
        bn, split = pins[key]
        return dict(kw, block_n=bn, split_k=split)

    def _wgrad_list(self):
        """How a whole layer's backward (_layer_backward, _ContextNode) launches its weight gradients: [] to gather them into grouped
        launches (ops.group_wgrad 1 and 3: the layer's four in one; 4: the FFN pair, then the attention pair), None for singles."""
        return [] if ops.group_wgrad in (1, 3, 4) else None

    def _layer_wgrad(self, sq, wg, i, key, dy, x, bias=False):
        """The weight gradient of layer i's linear key (out, inter, ao or qkv) from dy and its input x, on the side queue sq, with
        the bias column sum of dy when bias. wg None: launched now, pinned (_split_wgrad_kw). wg a list (_wgrad_list): the
        descriptor joins it and the bias sum runs now; the list goes out as one grouped launch at the layer's last weight
        gradient (QKV) and, in ops.group_wgrad 4, at the FFN's last (inter)."""
        li = self._lin["l%d.%s" % (i, key)]
        M = dy.shape[0]
        colsum = (lambda: ops.colsum(dy, li.gb, M, li.n)) if bias else None
        if wg is None:
            kw = self._split_wgrad_kw(key, li, dy, x, M)
            sq.run(lambda: (ops.gemm(**kw), colsum and colsum()), dy, x)
            return
        wg.append((self._wgrad_kw(li, dy, x, M), (dy, x)))
        if key == "qkv" or (key == "inter" and ops.group_wgrad == 4):
            self._issue_wgrads(sq, wg, colsum)
        elif colsum is not None:
            sq.run(colsum, dy)

    def _issue_wgrads(self, sq, wg, then=None):
        """The weight gradients gathered in wg (None: none) as one grouped launch on the side queue (a plain launch for one),
        followed by then(); wg is emptied."""
        if wg:
            kws = [kw for kw, _ in wg]
            sq.run(lambda: (ops.gemm_wgrad_group(kws), then and then()), *(t for _, keep in wg for t in keep))
            wg.clear()

    def _dgrad(self, li, dy, rows, out, **kw):
        ops.gemm(mode=ops.CB_GEMM_NN, m=rows, n=li.k, k=li.n, a=dy, a_rows=rows, a_ld=li.n, b=li.w, b_rows=li.n, b_ld=li.k,
                 out=out, out_ld=kw.pop("out_ld", li.k), **kw)

    def _mlp_head_backward(self, st, dlogits, nseq, H, tanh=True, grads=True):
        """Returns d pooler pre-activation (bf16, [nseq, H]); tanh = False: d pooled_output. grads = False: no parameter gradient
        is written."""
        dev = dlogits.device
        bf16 = torch.bfloat16
        c0, c2, pl = self._lin["cls0"], self._lin["cls2"], self._lin["pooler"]
        dl = torch.empty(nseq, c2.n, dtype=bf16, device=dev)
        ops.pad_cast(dlogits.float().contiguous() if dlogits.dtype != torch.float32 or not dlogits.is_contiguous() else dlogits, dl)
        if grads:
            self._wgrad(c2, dl, st["c1"], nseq)
            ops.colsum(dl, c2.gb, nseq, c2.n)
        dc1 = torch.empty(nseq, c0.n, dtype=bf16, device=dev)
        self._dgrad(c2, dl, nseq, dc1, aux=st["c1"], aux_ld=c0.n, aux_mode=ops.AUX_RELU_MASK)
        if grads:
            self._wgrad(c0, dc1, st["pd"], nseq)
            ops.colsum(dc1, c0.gb, nseq, c0.n)
        dpooled = torch.empty(nseq, H, dtype=bf16, device=dev)
        # d(pooler pre-activation) = (dc1 @ W0) * dropout_mask * tanh'(pooled)
        tanh_kw = dict(aux=st["pooled"], aux_ld=H, aux_mode=ops.AUX_TANH_GRAD) if tanh else {}
        self._dgrad(c0, dc1, nseq, dpooled, dropout_p=st["p_h"], dropout_seed=st["seed"] + 5, **tanh_kw)
        if self._capture is not None:
            self._capture.setdefault("bwd", {}).update(dl=dl, dc1=dc1)
        return dpooled

    def _head_backward(self, st, dout, nseq, H, tanh=True, grads=True):
        return self._mlp_head_backward(st, dout, nseq, H, tanh, grads)

    def _backward_impl(self, st, dout, grid_needs_grad):
        try:
            return self._backward_body(st, dout, grid_needs_grad)
        finally:
            ops.dropout_offset_bind(None)

    def _backward_body(self, st, dout, grid_needs_grad):
        self._flat.attach_grads()
        dev = st["x_last"].device
        H = _cfg(self.config, "hidden_size")
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        M = nseq * L
        ops.dropout_offset_bind(st.get("drop_word"))       # regenerate exactly this forward's masks
        cap = None if self._capture is None else self._capture.setdefault("bwd", {})
        sq = ops.SideQueue()                               # wgrad GEMMs / bias sums run beside the dgrad chain
        base = st.get("base_grads")                        # ClipBertBaseModel.forward: (d sequence, d pooled, d hidden states)
        dhidden = dattn = None
        ret_hidden, ret_attn = st.get("retained") or (None, None)   # outputs of ClipBertBaseModel.forward with retain_grad()
        if base is None:
            dpre = self._head_backward(st, dout, nseq, H)  # grad w.r.t. pooler pre-activation
        else:
            dpre, dseq, dhidden, dattn = self._base_output_grads(st, base, M, H)
        dx = self._pooler_backward(dpre, st["x_last"], nseq, L, H)
        extra = self._extra_sequence_grad(st) if base is None else dseq
        if cap is not None:      # clones where an add below writes the tensor in place
            cap.update(dpre=dpre, extra=extra, dx_pooler=dx.clone() if extra is not None or dhidden is not None else dx)
        if extra is not None:
            dx += extra
        for i in reversed(range(len(st["layers"]))):
            if dhidden is not None and dhidden[i + 1] is not None:     # output of layer i = hidden_states[i + 1]
                if cap is not None and i + 1 < len(st["layers"]):
                    cap["l%d" % (i + 1)]["dxn"] = dx.clone()
                dx += dhidden[i + 1]
            if ret_hidden is not None:
                _set_retained_hidden_grad(ret_hidden[i + 1], dx, nseq, L, H)
            ly = st["layers"][i]
            if ly.get("recompute"):
                # recompute_activations: the layer's forward re-run from its kept input under this pass's seeds and bound dropout
                # word (the forward's masks), beside the weight gradients of the layer above; then the join makes the main
                # stream wait for those, their activations' last readers, and drops them
                ly = self._recompute_layer(st, i, ly)
                sq.join()
            dx = self._layer_backward(st, i, ly, dx, sq, cap, None if dattn is None else dattn[i],
                                      None if ret_attn is None else ret_attn[i])
            st["layers"][i] = ly = None     # free this layer's stash
        if dhidden is not None and dhidden[0] is not None:                 # hidden_states[0] = the embedding output
            if cap is not None and len(st["layers"]):
                cap["l0"]["dxn"] = dx.clone()
            dx += dhidden[0]
        if ret_hidden is not None:
            _set_retained_hidden_grad(ret_hidden[0], dx, nseq, L, H)
        dgrid = self._embedding_backward(st, dx, grid_needs_grad)
        sq.join()          # every weight gradient is in the flat buffer before the caller (all-reduce hook, optimizer) sees it
        if cap is not None:
            cap.update(dx_emb=dx, dgrid=dgrid)
        if not self._optimizer_emits_packed:
            self._dirty = True
        return dgrid

    def _recompute_layer(self, st, i, ly):
        """Encoder layer i's stash as the forward kept it, from its kept input ly["x"]: the forward's launches, seeds and (bound by
        the caller) dropout word, so every tensor is the forward's bit for bit. The layer output is not needed."""
        stash, _, _ = self._layer_fwd(st, i, ly["x"], True, False)
        return dict(stash, seed=ly["seed"])

    def _pooler_backward(self, dpre, x_last, nseq, L, H, grads=True):
        """d pooler pre-activation (None: no gradient) -> the gradient at the top of the encoder, [nseq * L, H] bf16 with the [CLS]
        rows filled; grads: the pooler's weight and bias gradients into the flat buffer."""
        pl = self._lin["pooler"]
        if dpre is not None and grads:
            self._wgrad(pl, dpre, x_last, nseq, x_ld=L * H)
            ops.colsum(dpre, pl.gb, nseq, H)
        dx = torch.zeros(nseq * L, H, dtype=torch.bfloat16, device=x_last.device)
        if dpre is not None:
            self._dgrad(pl, dpre, nseq, dx, out_ld=L * H)  # scatters into the [CLS] rows
        return dx

    def _layer_backward(self, st, i, ly, dx, sq, cap=None, dattn=None, ret_attn=None, grads=True):
        """Encoder layer i from the gradient at its output dx ([nseq * L, H] bf16, not written) to the gradient at its input, with
        the layer's stash ly: the four per-module pieces in order, their weight gradients on the side queue sq as _wgrad_list
        says. dattn: a loss term on the layer's returned attention map, ret_attn: the map when retained. grads = False: no
        parameter gradient is written (a backward that does not accumulate into the parameters)."""
        c = None if cap is None else cap.setdefault("l%d" % i, {})
        wg = self._wgrad_list()
        du, ds2 = self._output_backward(st, i, ly, dx, sq, grads, fused=True, wg=wg, cap=c)
        da = self._intermediate_backward(st, i, ly, du, sq, grads, ds2, wg=wg)
        dctx, ds1 = self._self_output_backward(st, i, ly, da, sq, grads, wg=wg, cap=c)
        dxn = self._self_attention_backward(st, i, ly, dctx, dattn, sq, grads, ds1, wg=wg, cap=c, ret_attn=ret_attn)
        if c is not None:
            c.update(dx=dx, ds2=ds2, du=du, da=da, ds1=ds1, dctx=dctx)
            c.setdefault("dxn", dxn)
        return dxn

    def _map_backward(self, st, i, ly, G, handover, sq, grads=True):
        """The rest of encoder layer i's backward from G, the full gradient of its attention map (fp32 [nseq, heads, L, L]), when
        the backward is split at the map (_MapNode): dQ / dK written from G (cb_attention_probs_bwd_store), then the QKV tail.
        handover = (dqkv with its V block, ds1) from _ContextNode, or None when the layer's output got no gradient (dV = 0, no
        residual)."""
        nseq, _, _, _, _, lt, L = st["dims"]
        H, heads = st["H"], st["heads"]
        if handover is None:
            dqkv, ds1 = torch.empty(nseq * L, 3 * H, dtype=torch.bfloat16, device=G.device), None
            dqkv[:, 2 * H:].zero_()
        else:
            dqkv, ds1 = handover
        drow = torch.empty(nseq, heads, L, dtype=torch.float32, device=G.device)
        ops.attention_probs_bwd_store(ly["qkv"], st["mask"], ly["lse"], G, drow, dqkv, nseq, L, lt, heads, st["p_a"], ly["seed"] + 1)
        return self._qkv_backward(st, i, ly, dqkv, sq, grads, ds1, wg=[])

    # ---- the backward's per-module pieces: _layer_backward calls them in this order, the module path's split layers one by one -
    # wg: the layer's weight gradients, as _layer_wgrad takes them; cap: the layer's dict of captured gradients, or None
    def _output_backward(self, st, i, ly, dy, sq, grads, fused, wg=None, cap=None):
        """layer[i].output from the gradient dy at its output: (d intermediate_output, times gelu' when fused; ds2, the gradient
        of its residual input attention_output)."""
        M, H = dy.shape
        p_h, ls = st["p_h"], ly["seed"]
        in_l, out_l = self._lin["l%d.inter" % i], self._lin["l%d.out" % i]
        g2, _, dg2, db2 = self._ln("l%d.ln2" % i)
        dbo = out_l.gb
        if not grads:
            dg2 = db2 = dbo = None
        ds2 = torch.empty(M, H, dtype=torch.bfloat16, device=dy.device)
        ds2d = torch.empty_like(ds2) if p_h > 0 else None
        ops.layernorm_bwd(dy, ly["s2"], ly["st2"], g2, ds2, ds2d, dg2, db2, dbo, p_h, ls + 3)
        dd = ds2d if ds2d is not None else ds2
        if grads:
            self._layer_wgrad(sq, wg, i, "out", dd, ly["gel"])
        dgel = torch.empty(M, in_l.n, dtype=torch.bfloat16, device=dy.device)
        if fused:
            self._dgrad(out_l, dd, M, dgel, aux=ly["u"], aux_ld=in_l.n, aux_mode=ops.AUX_MUL)
        else:
            self._dgrad(out_l, dd, M, dgel)
        if cap is not None:
            cap["ds2d"] = ds2d
        return dgel, ds2

    def _intermediate_backward(self, st, i, ly, du, sq, grads, residual, wg=None):
        """layer[i].intermediate from du, the gradient at its pre-activation: d attention_output, plus residual (ds2) in the
        dgrad epilogue when given."""
        M, H = du.shape[0], st["H"]
        in_l = self._lin["l%d.inter" % i]
        if grads:
            self._layer_wgrad(sq, wg, i, "inter", du, ly["a"], bias=True)
        da = torch.empty(M, H, dtype=torch.bfloat16, device=du.device)
        if residual is None:
            self._dgrad(in_l, du, M, da)
        else:
            self._dgrad(in_l, du, M, da, residual=residual, res_ld=H)
        return da

    def _self_output_backward(self, st, i, ly, da, sq, grads, wg=None, cap=None):
        """layer[i].attention.output from the gradient da at its output: (d context, ds1 = the gradient of its residual input)."""
        M, H = da.shape
        p_h, ls = st["p_h"], ly["seed"]
        ao_l = self._lin["l%d.ao" % i]
        g1, _, dg1, db1 = self._ln("l%d.ln1" % i)
        dbao = ao_l.gb
        if not grads:
            dg1 = db1 = dbao = None
        ds1 = torch.empty(M, H, dtype=torch.bfloat16, device=da.device)
        ds1d = torch.empty_like(ds1) if p_h > 0 else None
        ops.layernorm_bwd(da, ly["s1"], ly["st1"], g1, ds1, ds1d, dg1, db1, dbao, p_h, ls + 2)
        dd1 = ds1d if ds1d is not None else ds1
        if grads:
            self._layer_wgrad(sq, wg, i, "ao", dd1, ly["ctx"])
        dctx = torch.empty(M, H, dtype=torch.bfloat16, device=da.device)
        self._dgrad(ao_l, dd1, M, dctx)
        if cap is not None:
            cap["ds1d"] = ds1d
        return dctx, ds1

    def _self_attention_backward(self, st, i, ly, dctx, dattn, sq, grads, residual, wg=None, cap=None, ret_attn=None):
        """layer[i].attention.self from d context (the forward's own context O in the attention backward) and dattn, a gradient
        of its map or None: the gradient at its input, plus residual (ds1) in the dgrad epilogue when given. ret_attn: the
        returned map when retained (its .grad gets dO V^T)."""
        nseq, _, _, _, _, lt, L = st["dims"]
        H, heads = st["H"], st["heads"]
        ls = ly["seed"]
        dqkv = torch.empty(nseq * L, 3 * H, dtype=torch.bfloat16, device=dctx.device)
        ops.attention_bwd(ly["qkv"], st["mask"], ly["ctx"], dctx, ly["lse"], dqkv, nseq, L, lt, heads, st["p_a"], ls + 1)
        if dattn is not None:      # a loss on attentions[i]: its dQ / dK added into dqkv
            drow = torch.empty(nseq, heads, L, dtype=torch.float32, device=dctx.device)
            if cap is not None:
                cap["dqkv_attn"] = dqkv.clone()
            ops.attention_probs_bwd(ly["qkv"], st["mask"], ly["lse"], dattn, drow, dqkv, nseq, L, lt, heads, st["p_a"], ls + 1)
        if ret_attn is not None:
            _add_retained_attention_grad(ret_attn, ly["qkv"], dctx, nseq, L, heads)
        if cap is not None:
            cap["dqkv"] = dqkv
        return self._qkv_backward(st, i, ly, dqkv, sq, grads, residual, wg)

    def _qkv_backward(self, st, i, ly, dqkv, sq, grads, residual, wg=None):
        """The QKV linear of layer[i].attention.self from dqkv: its weight gradient, the last of the layer, and the gradient at
        the layer input, plus residual (ds1) in the dgrad epilogue when given."""
        M, H = dqkv.shape[0], st["H"]
        qkv_l = self._lin["l%d.qkv" % i]
        if grads:
            self._layer_wgrad(sq, wg, i, "qkv", dqkv, ly["x"], bias=True)
        dxn = torch.empty(M, H, dtype=torch.bfloat16, device=dqkv.device)
        if residual is None:
            self._dgrad(qkv_l, dqkv, M, dxn)
        else:
            self._dgrad(qkv_l, dqkv, M, dxn, residual=residual, res_ld=H)
        return dxn

    def _embedding_backward(self, st, dx, grid_needs_grad, grads=True):
        """The text and visual embeddings from the gradient at their output dx; returns d visual_inputs (None unless
        grid_needs_grad). grads = False: no parameter gradient is written (the visual kernel's go to scratch)."""
        if grads:
            self._text_embedding_backward(st, st["ids"], dx)
        return self._visual_embedding_backward(st, st["grid"], st["repeat"], dx, grid_needs_grad, grads)

    def _text_embedding_backward(self, st, ids, dx):
        """bert.embeddings' parameter gradients from the gradient at the encoder input dx (its text rows are read)."""
        nseq, _, _, _, _, lt, L = st["dims"]
        g_t, _, dg_t, db_t = self._ln("emb.ln")
        (word, dword), (pos, dpos), (typ, dtyp) = self._emb("emb.word"), self._emb("emb.pos"), self._emb("emb.type")
        ops.embed_text_bwd(dx, ids, word, pos, typ, g_t, st["stats_t"], dword, dpos, dtyp, dg_t, db_t, nseq, lt, L, st["p_h"],
                           st["seed"] + 1)

    def _text_vectors_backward(self, st, vec, dx, grads):
        """bert.embeddings from the gradient at the encoder input dx when its word vectors came from word_embeddings: returns d vec
        (fp32 [B' * Lt, H]); grads = False: the parameter gradients go to scratch."""
        nseq, _, _, _, _, lt, L = st["dims"]
        g_t, _, dg_t, db_t = self._ln("emb.ln")
        (pos, dpos), (typ, dtyp) = self._emb("emb.pos"), self._emb("emb.type")
        if not grads:
            dpos, dtyp, dg_t, db_t = (torch.zeros_like(t) for t in (dpos, dtyp, dg_t, db_t))
        dvec = torch.empty(nseq * lt, vec.shape[1], dtype=torch.float32, device=dx.device)
        ops.embed_text_bwd_vectors(dx, vec, pos, typ, g_t, st["stats_t"], dvec, dpos, dtyp, dg_t, db_t, nseq, lt, L, st["p_h"],
                                   st["seed"] + 1)
        return dvec

    def _visual_embedding_backward(self, st, grid, repeat, dx, grid_needs_grad, grads=True):
        """bert.visual_embeddings from the gradient at the encoder input dx (its visual rows are read); returns d grid (None
        unless grid_needs_grad)."""
        dev = dx.device
        H = _cfg(self.config, "hidden_size")
        nseq, _, T, gh, gw, lt, L = st["dims"]
        nvid = grid.shape[0]
        p_h = st["p_h"]
        bf16 = torch.bfloat16
        n_ex, s2v, starts = repeat
        g_v, _, dg_v, db_v = self._ln("vis.ln")
        (row, drow), (col, dcol), (vtyp, dvtyp) = self._emb("vis.row"), self._emb("vis.col"), self._emb("vis.type")
        if not grads:
            if not grid_needs_grad:
                return None
            drow, dcol, dvtyp, dg_v, db_v = (torch.zeros_like(t) for t in (drow, dcol, dvtyp, dg_v, db_v))
        dv_tmp = torch.empty(nseq * gh * gw, H, dtype=torch.float32, device=dev)
        dgrid = torch.empty(nvid, T, gh, gw, H, dtype=bf16, device=dev) if grid_needs_grad else None
        sample = st.get("sample")
        if sample is None:
            ops.embed_visual_bwd(dx, grid, s2v, starts, n_ex, row, col, vtyp, g_v, st["stats_v"], dv_tmp, dgrid, drow, dcol, dvtyp,
                                 dg_v, db_v, nseq, nvid, T, gh, gw, lt, L, p_h, st["seed"] + 2)
        else:
            # sampled visual tokens (see _forward_impl): gradients of the (n_keep x 1) virtual grid, scattered back by index
            idx, gh0, gw0, row_s, col_s = sample
            drow_s, dcol_s = torch.zeros_like(row_s), torch.zeros_like(col_s)
            ops.embed_visual_bwd(dx, grid, s2v, starts, n_ex, row_s, col_s, vtyp, g_v, st["stats_v"], dv_tmp, dgrid, drow_s, dcol_s,
                                 dvtyp, dg_v, db_v, nseq, nvid, T, gh, gw, lt, L, p_h, st["seed"] + 2)
            if grads:
                drow.index_add_(0, idx // gw0, drow_s)         # d(row[r] + col[c]) goes to both tables
                dcol.index_add_(0, idx % gw0, drow_s)
            if dgrid is not None:
                full = torch.zeros(nvid, T, gh0 * gw0, H, dtype=bf16, device=dev)
                full.index_copy_(2, idx, dgrid.view(nvid, T, gh, H))
                dgrid = full.view(nvid, T, gh0, gw0, H)
        return dgrid

    def _extra_sequence_grad(self, st):
        return None

    def _base_output_grads(self, st, grads, M, H):
        """Upstream gradients of ClipBertBaseModel.forward -> (d pooler pre-activation or None, dense d sequence_output or None,
        [d hidden_states[k] or None] or None, [d attentions[k] or None] or None), bf16 but the attention gradients (contiguous
        fp32: an expanded gradient such as the one of attn.sum() is materialised). d pooled goes through tanh' = 1 - pooled^2
        (BertPooler, transformers.py:470-476) as the heads' dpre does, here as one product on the (B', 768) rows."""
        dseq, dpooled, dh, da = grads
        bf16 = torch.bfloat16

        def dense(g):
            return None if g is None else g.reshape(M, H).to(bf16).contiguous()

        dpre = None if dpooled is None else _pooler_pre_grad(st["pooled"], dpooled)
        dattn = None
        if any(g is not None for g in da):
            dattn = [None if g is None else g.to(torch.float32).contiguous() for g in da]
        return dpre, dense(dseq), ([dense(g) for g in dh] if dh else None), dattn

    # ---- misc -------------------------------------------------------------------------------------
    def zero_grad(self, set_to_none=False):
        if self._flat is not None and self._flat.grad is not None:
            self._flat.zero_grad()
        else:
            super().zero_grad(set_to_none=set_to_none)


def _pooler_pre_grad(pooled, dpooled):
    """d pooler pre-activation (bf16) = d pooled * tanh' = d pooled (1 - pooled^2), as one product on the (B', 768) rows."""
    p = pooled.float()
    return (dpooled.float() * (1.0 - p * p)).to(torch.bfloat16)


def _set_retained_hidden_grad(tensors, dx, nseq, L, H):
    """.grad of a retained hidden state (or sequence_output) = dx, the full gradient at that layer boundary: it already holds
    the direct term the retain hook put in .grad, and the backward writes dx no more after this point, so it is not copied."""
    for t in tensors:
        t.grad = dx.view(nseq, L, H)


def _add_retained_attention_grad(t, qkv, dctx, nseq, L, heads):
    """attentions[i].grad (+)= dO V^T, the term the returned map receives from the context product, by cb_attention_dprobs:
    added in place to the direct term the retain hook left in .grad, or written into a fresh tensor when there is none (or
    when .grad is not a contiguous, 16-byte aligned tensor, which is then copied first)."""
    g = t.grad
    if g is not None and g.is_contiguous() and g.data_ptr() % 16 == 0:
        ops.attention_dprobs(qkv, dctx, g, True, nseq, L, heads)
        return
    out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
    if g is not None:
        out.copy_(g)
    ops.attention_dprobs(qkv, dctx, out, g is not None, nseq, L, heads)
    t.grad = out


class _BaseModelEngine(_ClipBertHeadModel):
    """The engine of a ClipBertBaseModel constructed on its own: flat storage for the base model's parameters, no head. It is
    reached through the base model's back-reference only, so its own training flag is never read (base passes use bert's)."""

    def __init__(self, config, bert):
        super().__init__(config, bert=bert)

    def _head_linears(self):
        return []


class _MlpHeadMixin:
    def _make_classifier(self, config, num_out):
        h = _cfg(config, "hidden_size")
        self.classifier = nn.Sequential(nn.Linear(h, h * 2), nn.ReLU(True), nn.Linear(h * 2, num_out))

    def _head_linears(self):
        return [("cls0", self.classifier[0]), ("cls2", self.classifier[2])]


class ClipBertForVideoTextRetrieval(_MlpHeadMixin, _ClipBertHeadModel):
    """src/modeling/modeling.py:523-580."""

    def __init__(self, config):
        super().__init__(config)
        self._make_classifier(config, _cfg(config, "num_labels"))
        self.margin = _cfg(config, "margin", 0.2)
        _init_bert_weights(self, _cfg(config, "initializer_range", 0.02))

    def _num_head_outputs(self):
        return _cfg(self.config, "num_labels")

    def forward(self, text_input_ids, visual_inputs, text_input_mask, labels=None, sample_size=-1, _repeat_counts=None):
        logits = self._run(text_input_ids, visual_inputs, text_input_mask, _repeat_counts)
        logits, loss = self.calc_loss(logits, labels, sample_size=sample_size)
        return dict(logits=logits, loss=loss)

    def calc_loss(self, logits, labels, sample_size=-1):
        if labels is None:
            return logits, 0
        loss_type = _cfg(self.config, "loss_type")
        if loss_type == "ce":
            loss = cross_entropy_none(logits.view(-1, _cfg(self.config, "num_labels")), labels.view(-1))
        elif loss_type == "rank":
            scores = torch.sigmoid(logits).squeeze()
            assert sample_size > 0
            scores = scores.contiguous().view(sample_size, -1)
            loss = torch.clamp(self.margin + scores[:, 1:] - scores[:, :1], min=0)
        else:
            raise ValueError("Invalid option for config.loss_type")
        return logits, loss


class _CrossEntropyNone(torch.autograd.Function):
    """``F.cross_entropy(logits, labels, reduction="none")`` on cb_cross_entropy_fwd / _bwd: one pass over each row forward, one
    backward (ATen materialises a log-softmax of the size of the logits - 30 522 columns for the masked-LM loss)."""

    @staticmethod
    def forward(ctx, logits, labels):
        z = logits.detach()
        if z.dtype != torch.float32 or z.stride(-1) != 1:
            z = z.float().contiguous()
        y = labels.to(torch.int64).contiguous()
        loss = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        lse = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        ops.cross_entropy_fwd(z, y, loss, lse)
        ctx.save_for_backward(z, y, lse)
        ctx.in_dtype = logits.dtype
        return loss

    @staticmethod
    def backward(ctx, g):
        z, y, lse = ctx.saved_tensors
        dz = torch.empty_like(z)
        ops.cross_entropy_bwd(z, y, lse, g.to(torch.float32).contiguous(), dz)
        return dz.to(ctx.in_dtype), None


def cross_entropy_none(logits, labels):
    """The reference's ``F.cross_entropy(..., reduction="none")`` calls (src/modeling/modeling.py:286-299,430-436,560-566) on this
    library's kernel for CUDA tensors; ``logits`` (rows, C), ``labels`` (rows,) with ignore_index -100."""
    _require_cuda(logits)
    return _CrossEntropyNone.apply(logits, labels)


def instance_bce_with_logits(logits, labels, reduction="mean"):
    """src/modeling/modeling.py:310-316."""
    assert logits.dim() == 2
    loss = F.binary_cross_entropy_with_logits(logits, labels, reduction=reduction)
    if reduction == "mean":
        loss *= labels.size(1)
    return loss


class ClipBertForSequenceClassification(_MlpHeadMixin, _ClipBertHeadModel):
    """src/modeling/modeling.py:327-384."""

    def __init__(self, config):
        super().__init__(config)
        self._make_classifier(config, _cfg(config, "num_labels"))
        _init_bert_weights(self, _cfg(config, "initializer_range", 0.02))

    def _num_head_outputs(self):
        return _cfg(self.config, "num_labels")

    def forward(self, text_input_ids, visual_inputs, text_input_mask, labels=None, _repeat_counts=None, **_unused):
        logits = self._run(text_input_ids, visual_inputs, text_input_mask, _repeat_counts)
        logits, loss = self.calc_loss(logits, labels)
        return dict(logits=logits, loss=loss)

    def calc_loss(self, logits, labels):
        if labels is None:
            return logits, 0
        nl = _cfg(self.config, "num_labels")
        if nl == 1:
            loss = F.mse_loss(logits.view(-1), labels.view(-1), reduction="none")
        elif _cfg(self.config, "loss_type") == "bce":
            loss = instance_bce_with_logits(logits, labels, reduction="none")
        elif _cfg(self.config, "loss_type") == "ce":
            loss = cross_entropy_none(logits.view(-1, nl), labels.view(-1))
        else:
            raise ValueError("Invalid option for config.loss_type")
        return logits, loss


class ClipBertForMultipleChoice(_MlpHeadMixin, _ClipBertHeadModel):
    """src/modeling/modeling.py:387-451 — one score per (video, option); CE over options."""

    def __init__(self, config):
        super().__init__(config)
        self._make_classifier(config, 1)
        _init_bert_weights(self, _cfg(config, "initializer_range", 0.02))

    def _num_head_outputs(self):
        return 1

    def forward(self, text_input_ids, visual_inputs, text_input_mask, labels=None, _repeat_counts=None, **_unused):
        logits = self._run(text_input_ids, visual_inputs, text_input_mask, _repeat_counts)
        logits, loss = self.calc_loss(logits, labels)
        return dict(logits=logits, loss=loss)

    def calc_loss(self, logits, labels):
        nl = _cfg(self.config, "num_labels")
        loss_type = _cfg(self.config, "loss_type")
        if loss_type == "ce":
            logits = logits.reshape(-1, nl)
        if labels is None:
            return logits, 0
        if nl == 1:
            loss = F.mse_loss(logits.view(-1), labels.view(-1), reduction="none")
        elif loss_type == "bce":
            loss = instance_bce_with_logits(logits, labels, reduction="none")
        elif loss_type == "ce":
            loss = cross_entropy_none(logits, labels.view(-1))
        else:
            raise ValueError("Invalid option for config.loss_type")
        return logits, loss


class ClipBertForRegression(nn.Module):
    """src/modeling/modeling.py:454-507. The reference's task scripts import this name (run_video_qa.py:7-10,
    e2e_model.py:1-6) but never instantiate it - no task configuration selects it - so only the name exists here: its
    ELU + BatchNorm1d regressor has no kernels on this path, and constructing it says so instead of running something else."""

    def __init__(self, config):
        super().__init__()
        raise NotImplementedError("ClipBertForRegression is not built on the H100 path (unused by every reference task script)")


class BertPredictionHeadTransform(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.dense = nn.Linear(h, h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))


class BertLMPredictionHead(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(_cfg(config, "hidden_size"), _cfg(config, "vocab_size"), bias=False)
        self.bias = nn.Parameter(torch.zeros(_cfg(config, "vocab_size")))
        self.decoder.bias = self.bias          # hf 2.11 link (transformers.py:503-507)


class BertPreTrainingHeads(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.predictions = BertLMPredictionHead(config)
        self.seq_relationship = nn.Linear(_cfg(config, "hidden_size"), 2)


class ClipBertForPreTraining(_ClipBertHeadModel):
    """src/modeling/modeling.py:241-307 — MLM head on the text positions (tied decoder, vocab 30522) + ITM head.

    Head kernels: strided gather of the text rows, cb_gemm(+bias, GELU, stash) -> cb_layernorm_fwd ->
    cb_gemm against the bf16 copy of the word table (N padded 30522 -> 30528, fp32 logits) ; ITM = cb_gemm on
    the pooled output. The per-token CE (ignore_index -100) stays torch glue on the returned logits.
    """

    def __init__(self, config):
        super().__init__(config)
        self.cls = BertPreTrainingHeads(config)
        _init_bert_weights(self, _cfg(config, "initializer_range", 0.02))
        self.cls.predictions.decoder.weight = self.bert.embeddings.word_embeddings.weight      # tied (get_output_embeddings)
        self._word_bf16 = None

    def _head_linears(self):
        return [("itm", self.cls.seq_relationship), ("mlm_t", self.cls.predictions.transform.dense)]

    def _extra_layernorms(self):
        return [("mlm_ln", self.cls.predictions.transform.LayerNorm)]

    def _extra_params(self):
        v = self.cls.predictions.bias.shape[0]
        return [("mlm_bias", self.cls.predictions.bias, (v + 7) // 8 * 8)]

    def _num_head_outputs(self):
        return 2

    @torch.no_grad()
    def _repack(self):
        super()._repack()
        e = self._spec["emb.word"]
        v, h = e["param"].shape
        vp = (v + 7) // 8 * 8
        if self._word_bf16 is None or self._word_bf16.device != self._flat.master.device:
            self._word_bf16 = torch.zeros(vp, h, dtype=torch.bfloat16, device=self._flat.master.device)
        ops.cast_scale(self._flat.master[e["offset"]: e["offset"] + v * h], self._word_bf16.view(-1)[: v * h])

    def packed_written_by_optimizer(self):
        super().packed_written_by_optimizer()
        e = self._spec["emb.word"]                 # the tied MLM decoder reads a bf16 copy of the word-embedding table
        v, h = e["param"].shape
        if self._word_bf16 is not None:
            ops.cast_scale(self._flat.master[e["offset"]: e["offset"] + v * h], self._word_bf16.view(-1)[: v * h])

    def _head_forward(self, pooled, st, nseq, p_h, seed, need_backward):
        dev = pooled.device
        H = pooled.shape[1]
        nseq_, nvid, T, gh, gw, lt, L = st["dims"]
        bf16 = torch.bfloat16
        itm_l, t_l = self._lin["itm"], self._lin["mlm_t"]
        itm = torch.empty(nseq, itm_l.n, dtype=torch.float32, device=dev)
        self._gemm_fwd(pooled, nseq, itm_l, itm, out_fp32=1)
        # text rows of the final sequence output (sequence_output[:, :txt_len], modeling.py:283-285)
        R = nseq * lt
        xt = st["x_last"].view(nseq, L, H)[:, :lt].contiguous().view(R, H)
        u = torch.empty(R, H, dtype=bf16, device=dev)
        t1 = torch.empty(R, H, dtype=bf16, device=dev)
        self._gemm_fwd(xt, R, t_l, t1, act=ops.ACT_GELU, out2=u, out2_ld=H)
        g, b, _, _ = self._ln("mlm_ln")
        t2 = torch.empty(R, H, dtype=bf16, device=dev)
        stats = torch.empty(R, 2, dtype=torch.float32, device=dev)
        ops.layernorm_fwd(t1, g, b, t2, stats, float(_cfg(self.config, "layer_norm_eps")))
        e = self._spec["mlm_bias"]
        vp = self._word_bf16.shape[0]
        bias = self._flat.master[e["offset"]: e["offset"] + vp]
        scores = torch.empty(R, vp, dtype=torch.float32, device=dev)
        ops.gemm(mode=ops.CB_GEMM_TN, m=R, n=vp, k=H, a=t2, a_rows=R, a_ld=H, b=self._word_bf16, b_rows=vp, b_ld=H, shift=bias,
                 out=scores, out_ld=vp, out_fp32=1)
        st.update(xt=xt, mlm_u=u, mlm_t1=t1, mlm_t2=t2, mlm_stats=stats)
        if self._capture is not None:
            self._capture.update(itm=itm, xt=xt, mlm_u=u, t1=t1, t2=t2, mlm_stats=stats, scores=scores)
        v = _cfg(self.config, "vocab_size")
        return itm[:, :2], scores.view(nseq, lt, vp)[:, :, :v]

    def _head_backward(self, st, douts, nseq, H, tanh=True, grads=True):
        ditm, dscores = douts
        dev = st["x_last"].device
        bf16 = torch.bfloat16
        nseq_, nvid, T, gh, gw, lt, L = st["dims"]
        R = nseq * lt
        itm_l, t_l = self._lin["itm"], self._lin["mlm_t"]
        cap = None if self._capture is None else self._capture.setdefault("bwd", {})
        dpre = torch.zeros(nseq, H, dtype=bf16, device=dev)
        if ditm is not None:
            dl = torch.empty(nseq, itm_l.n, dtype=bf16, device=dev)
            ops.pad_cast(ditm.float().contiguous(), dl)
            if grads:
                self._wgrad(itm_l, dl, st["pooled"], nseq)
                ops.colsum(dl, itm_l.gb, nseq, itm_l.n)
            self._dgrad(itm_l, dl, nseq, dpre, **(dict(aux=st["pooled"], aux_ld=H, aux_mode=ops.AUX_TANH_GRAD) if tanh else {}))
            if cap is not None:
                cap["dl"] = dl
        st["mlm_dx"] = None
        if dscores is not None:
            vp = self._word_bf16.shape[0]
            v = _cfg(self.config, "vocab_size")
            ds = torch.empty(R, vp, dtype=bf16, device=dev)
            ops.pad_cast(dscores.reshape(R, v).float().contiguous(), ds)
            e = self._spec["emb.word"]
            gword = self._flat.grad[e["offset"]: e["offset"] + vp * H].view(vp, H)
            eb = self._spec["mlm_bias"]
            if grads:
                ops.gemm(mode=ops.CB_GEMM_WGRAD, m=vp, n=H, k=R, a=ds, a_rows=R, a_ld=vp, b=st["mlm_t2"], b_rows=R, b_ld=H, out=gword,
                         out_ld=H, out_fp32=1)
                ops.colsum(ds, self._flat.grad[eb["offset"]: eb["offset"] + vp], R, vp)
            dt2 = torch.empty(R, H, dtype=bf16, device=dev)
            ops.gemm(mode=ops.CB_GEMM_NN, m=R, n=H, k=vp, a=ds, a_rows=R, a_ld=vp, b=self._word_bf16, b_rows=vp, b_ld=H, out=dt2, out_ld=H)
            g, _, dg, db = self._ln("mlm_ln")
            if not grads:
                dg = db = None
            dt1 = torch.empty(R, H, dtype=bf16, device=dev)
            ops.layernorm_bwd(dt2, st["mlm_t1"], st["mlm_stats"], g, dt1, None, dg, db, None, 0.0, 0)
            # d(pre-GELU) = dt1 * gelu'(u): a dgrad-style epilogue needs a GEMM, so fold it into the dgrad of transform.dense
            # by first masking dt1 (relu_mask has no gelu form) -> use the NN GEMM of the *identity-free* path below
            du = torch.empty(R, H, dtype=bf16, device=dev)
            _gelu_bwd(dt1, st["mlm_u"], du)
            if grads:
                self._wgrad(t_l, du, st["xt"], R)
                ops.colsum(du, t_l.gb, R, H)
            dxt = torch.empty(R, H, dtype=bf16, device=dev)
            self._dgrad(t_l, du, R, dxt)
            st["mlm_dx"] = dxt
            if cap is not None:
                cap.update(ds=ds, dt2=dt2, dt1=dt1, mlm_du=du, dxt=dxt)
        return dpre

    def _extra_sequence_grad(self, st):
        dxt = st.get("mlm_dx")
        if dxt is None:
            return None
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        H = dxt.shape[1]
        full = torch.zeros(nseq, L, H, dtype=dxt.dtype, device=dxt.device)
        full[:, :lt] = dxt.view(nseq, lt, H)
        return full.view(nseq * L, H)

    def forward(self, text_input_ids, visual_inputs, text_input_mask, mlm_labels=None, itm_labels=None, _repeat_counts=None, **_unused):
        itm_scores, mlm_scores = self._run(text_input_ids, visual_inputs, text_input_mask, _repeat_counts)
        v = _cfg(self.config, "vocab_size")
        mlm_loss = cross_entropy_none(mlm_scores.reshape(-1, v), mlm_labels.view(-1)) if mlm_labels is not None else 0
        itm_loss = cross_entropy_none(itm_scores.view(-1, 2), itm_labels.view(-1)) if itm_labels is not None else 0
        return dict(mlm_scores=mlm_scores, mlm_loss=mlm_loss, mlm_labels=mlm_labels, itm_scores=itm_scores, itm_loss=itm_loss,
                    itm_labels=itm_labels)


def _gelu_bwd(dy, u, out):
    """out = dy * gelu'(u) for the MLM transform (BertPredictionHeadTransform, transformers.py:486-495): an elementwise kernel
    on one [R, 768] tensor - the GEMM that follows reads it as an operand, so no epilogue can carry this product."""
    ops.gelu_bwd(dy, u, out)
