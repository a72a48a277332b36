"""Cross-modal transformer half of ClipBERT on H100.

Mirrors the reference classes in ``src/modeling/modeling.py`` / ``src/modeling/transformers.py``
(ClipBertBaseModel, ClipBertForVideoTextRetrieval, ClipBertForSequenceClassification,
ClipBertForMultipleChoice, ClipBertForPreTraining): same constructor (a BertConfig-like object),
same forward signatures and return dicts, same state_dict keys (SURVEY.md App. B). The torch.nn
modules below are PARAMETER CONTAINERS only — their own ``forward`` is never called. All arithmetic
is the hand-written sm_90a kernels behind libclipbert_sm90.so:

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
class BertEmbeddings(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.word_embeddings = nn.Embedding(_cfg(config, "vocab_size"), h, padding_idx=_cfg(config, "pad_token_id", 0))
        self.position_embeddings = nn.Embedding(_cfg(config, "max_position_embeddings"), h)
        self.token_type_embeddings = nn.Embedding(_cfg(config, "type_vocab_size"), h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))


class VisualInputEmbedding(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.position_embeddings = nn.Embedding(_cfg(config, "max_position_embeddings"), h)   # unused (modeling.py:97)
        self.row_position_embeddings = nn.Embedding(_cfg(config, "max_grid_row_position_embeddings"), h)
        self.col_position_embeddings = nn.Embedding(_cfg(config, "max_grid_col_position_embeddings"), h)
        self.token_type_embeddings = nn.Embedding(1, h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))


class BertSelfAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.query, self.key, self.value = nn.Linear(h, h), nn.Linear(h, h), nn.Linear(h, h)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.dense = nn.Linear(h, h)
        self.LayerNorm = nn.LayerNorm(h, eps=_cfg(config, "layer_norm_eps"))


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(_cfg(config, "hidden_size"), _cfg(config, "intermediate_size"))


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(_cfg(config, "intermediate_size"), _cfg(config, "hidden_size"))
        self.LayerNorm = nn.LayerNorm(_cfg(config, "hidden_size"), eps=_cfg(config, "layer_norm_eps"))


class BertLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)


class BertEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.layer = nn.ModuleList([BertLayer(config) for _ in range(_cfg(config, "num_hidden_layers"))])


class BertPooler(nn.Module):
    def __init__(self, config):
        super().__init__()
        h = _cfg(config, "hidden_size")
        self.dense = nn.Linear(h, h)


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
    ``model.layerwise_autograd = True`` (default False; also on ``head.bert``) makes a pass that records autograd a chain of
    nodes - the embeddings, one node per encoder layer (two when the maps are differentiable: A_k, hidden_states[k] ->
    attentions[k], and C_k, (hidden_states[k], attentions[k]) -> hidden_states[k + 1], the reference's dataflow) and the
    pooler - with sequence_output the same tensor as hidden_states[12]. Tensor hooks, ``torch.autograd.grad``,
    ``retain_grad()`` and ``backward(inputs=...)`` on any map or hidden state then follow torch's semantics, and a hook that
    rewrites a map's gradient changes every gradient below that layer. Parameter gradients too: a node writes them only when
    the backward accumulates into the parameters (``autograd.grad`` leaves the flat gradient buffer as it was), and
    ``retain_graph=True`` allows a second backward. The forward issues the launches of the default; so does the backward of a
    layer whose map is not differentiable. Refused together with the overlapped data-parallel exchange
    (``enable_overlapped_allreduce``): the switch is for analysis, not training.
    """

    differentiable_attentions = False
    layerwise_autograd = False

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
        return self._engine._run_base(text_input_ids, visual_inputs, attention_mask, self.output_hidden_states, self.output_attentions,
                                      self.differentiable_attentions, self.layerwise_autograd)


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


class _LayerwisePass:
    """What the nodes of one layerwise bert(...) pass share: the engine, the pass's stash (its per-layer activations move into the
    nodes' saved tensors) and the hand-over from C_k to A_k of a map-split layer (dqkv with its V block, ds1)."""

    def __init__(self, module, st):
        self.module, self.st, self.handover = module, st, {}

    def dims(self):
        nseq, _, _, _, _, _, L = self.st["dims"]
        return nseq, L, _cfg(self.module.config, "hidden_size")

    def dense(self, g):
        """An upstream gradient of a hidden state as the engine's [nseq * L, H] contiguous bf16 operand."""
        nseq, L, H = self.dims()
        return g.reshape(nseq * L, H).to(torch.bfloat16).contiguous()

    def hidden(self, i):
        """hidden_states[i] as a fresh view: the input of layer i, or the top of the encoder."""
        nseq, L, H = self.dims()
        layers = self.st["layers"]
        return (layers[i]["x"] if i < len(layers) else self.st["x_last"]).view(nseq, L, H)


def _will_execute(ctx, k):
    """Whether the engine runs, in the current backward, the node behind tensor input k of this node (False when that input
    takes no gradient). For a parameter anchor: whether this backward accumulates into the parameters - backward() does;
    torch.autograd.grad() and backward(inputs=...) without the parameter do not."""
    node = ctx.next_functions[k][0]
    if node is None:
        return False
    try:
        return bool(torch._C._will_engine_execute_node(node))
    except RuntimeError:        # autograd.grad() with the anchor parameter among its inputs: no accumulation into .grad
        return False


class _EmbeddingNode(torch.autograd.Function):
    """(visual_inputs, anchor) -> hidden_states[0]."""

    @staticmethod
    def forward(ctx, ps, grid, anchor):
        st = ps.st
        ctx.ps = ps
        ctx.save_for_backward(st.pop("ids"), st.pop("grid"), st.pop("stats_t"), st.pop("stats_v"))
        return ps.hidden(0)

    @staticmethod
    def backward(ctx, dh):
        ids, grid, stats_t, stats_v = ctx.saved_tensors
        ps = ctx.ps
        grads, need_grid = _will_execute(ctx, 1), _will_execute(ctx, 0)
        if not (grads or need_grid):
            return None, None, None
        st = dict(ps.st, ids=ids, grid=grid, stats_t=stats_t, stats_v=stats_v)
        with ps.module._node_backward(st, grads):
            dgrid = ps.module._embedding_backward(st, ps.dense(dh), need_grid, grads)
        return None, dgrid, None


class _LayerNode(torch.autograd.Function):
    """Encoder layer i, hidden_states[i] -> hidden_states[i + 1] (maps not differentiable)."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        ly = ps.st["layers"][i]
        ctx.ps, ctx.i, ctx.seed = ps, i, ly["seed"]
        ctx.save_for_backward(*(ly[k] for k in _LAYER_STASH))
        return ps.hidden(i + 1)

    @staticmethod
    def backward(ctx, dy):
        ly = dict(zip(_LAYER_STASH, ctx.saved_tensors), seed=ctx.seed)
        ps, grads = ctx.ps, _will_execute(ctx, 1)
        with ps.module._node_backward(ps.st, grads) as sq:
            dxn = ps.module._layer_backward(ps.st, ctx.i, ly, ps.dense(dy), sq, grads=grads)
        return None, None, dxn.view(*ps.dims()), None


class _MapNode(torch.autograd.Function):
    """A_k: hidden_states[k] -> attentions[k]. Its backward receives the map's full gradient G (the direct term, C_k's dO V^T and
    whatever hooks made of them) and finishes layer k: dQ / dK from G, the QKV weight gradient, the dgrad to hidden_states[k]."""

    @staticmethod
    def forward(ctx, ps, i, h, anchor):
        ly = ps.st["layers"][i]
        ctx.ps, ctx.i, ctx.seed = ps, i, ly["seed"]
        ctx.save_for_backward(ly["x"], ly["qkv"], ly["lse"])
        return ps.st["attn"][i]

    @staticmethod
    def backward(ctx, G):
        x, qkv, lse = ctx.saved_tensors
        ps, grads = ctx.ps, _will_execute(ctx, 1)
        handover = ps.handover.pop(ctx.i, None)
        with ps.module._node_backward(ps.st, grads) as sq:
            dxn = ps.module._map_backward(ps.st, ctx.i, dict(x=x, qkv=qkv, lse=lse, seed=ctx.seed), G.to(torch.float32).contiguous(),
                                          handover, sq, grads)
        return None, None, dxn.view(*ps.dims()), None


class _ContextNode(torch.autograd.Function):
    """C_k: (hidden_states[k], attentions[k]) -> hidden_states[k + 1], the reference's dataflow past the map (ctx = A V, output
    projection, LN1, FFN, LN2). Its backward returns d A = dO V^T for the map and nothing for hidden_states[k]: dV and the
    residual ds1 are handed to A_k, which produces the whole gradient at hidden_states[k]."""

    @staticmethod
    def forward(ctx, ps, i, h, a, anchor):
        ly = ps.st["layers"][i]
        ctx.ps, ctx.i, ctx.seed = ps, i, ly["seed"]
        ctx.save_for_backward(*(ly[k] for k in _LAYER_STASH))
        return ps.hidden(i + 1)

    @staticmethod
    def backward(ctx, dy):
        ly = dict(zip(_LAYER_STASH, ctx.saved_tensors), seed=ctx.seed)
        ps, grads = ctx.ps, _will_execute(ctx, 2)
        split = "with_map" if _will_execute(ctx, 1) else "map_only"       # A_k runs in this backward: hand dV and ds1 over
        with ps.module._node_backward(ps.st, grads) as sq:
            dmap, handover = ps.module._layer_backward(ps.st, ctx.i, ly, ps.dense(dy), sq, grads=grads, split=split)
        if handover is not None:
            ps.handover[ctx.i] = handover
        return None, None, None, dmap, None


class _PoolerNode(torch.autograd.Function):
    """hidden_states[-1] (= sequence_output) -> pooled_output."""

    @staticmethod
    def forward(ctx, ps, h, anchor):
        ctx.ps = ps
        pooled = ps.st.pop("pooled")
        ctx.save_for_backward(ps.st.pop("x_last"), pooled)
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        x_last, pooled = ctx.saved_tensors
        ps, grads = ctx.ps, _will_execute(ctx, 1)
        nseq, L, H = ps.dims()
        with ps.module._node_backward(ps.st, grads):
            dx = ps.module._pooler_backward(_pooler_pre_grad(pooled, dpooled), x_last, nseq, L, H, grads)
        return None, dx.view(nseq, L, H), None


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

    def _run_base(self, text_input_ids, visual_inputs, attention_mask, want_hidden, want_attn, diff_attn=False, layerwise=False):
        """ClipBertBaseModel.forward on this engine (the head itself is not run). visual_inputs: (B', T, h, w, 768)."""
        _require_cuda(text_input_ids)
        self._ensure_ready(text_input_ids.device)
        assert visual_inputs.shape[0] == text_input_ids.shape[0], "visual_inputs must have one row per text example"
        grid = visual_inputs if visual_inputs.dtype == torch.bfloat16 else visual_inputs.to(torch.bfloat16)
        grid = grid.contiguous()
        ids = text_input_ids.contiguous()
        mask = attention_mask.to(torch.int64).contiguous()
        flags = (bool(want_hidden), bool(want_attn), bool(want_attn and diff_attn))
        if torch.is_grad_enabled() and (grid.requires_grad or any(p.requires_grad for p in self.bert.parameters())) and layerwise:
            seq, pooled, hidden, attn = self._run_layerwise(ids, grid, mask, flags)
        elif torch.is_grad_enabled() and (grid.requires_grad or any(p.requires_grad for p in self.bert.parameters())):
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

    def _run_layerwise(self, ids, grid, mask, flags):
        """ClipBertBaseModel.forward with layerwise_autograd: the pass runs as _forward_impl runs it (same launches, same bits),
        then its outputs are handed out through a chain of autograd nodes - the embeddings, one node per encoder layer (two, A_k
        and C_k, when the maps are differentiable) and the pooler - so that tensor hooks, torch.autograd.grad and
        backward(inputs=...) on any hidden state or map follow torch's own semantics. Returns (sequence_output, pooled_output,
        hidden_states, attentions) as _forward_impl does."""
        if self._grad_ready_hook is not None:
            raise RuntimeError("ClipBertBaseModel.layerwise_autograd is for analysis, not data-parallel training: it cannot run while "
                               "the overlapped gradient exchange (enable_overlapped_allreduce) is enabled")
        with torch.no_grad():
            (_, _, _, attn), st = self._forward_impl(ids, grid, mask, (1, None, None), need_backward=True, base=flags)
        st["attn"] = attn
        ps = _LayerwisePass(self, st)
        bert = self.bert
        h = _EmbeddingNode.apply(ps, grid, bert.embeddings.word_embeddings.weight)
        hidden, maps = [h], []
        for i, layer in enumerate(bert.encoder.layer):
            if flags[2]:
                a = _MapNode.apply(ps, i, h, layer.attention.self.query.weight)
                h = _ContextNode.apply(ps, i, h, a, layer.attention.output.dense.weight)
                maps.append(a)
            else:
                h = _LayerNode.apply(ps, i, h, layer.attention.self.query.weight)
            hidden.append(h)
        pooled = _PoolerNode.apply(ps, h, bert.pooler.dense.weight)
        st["layers"] = st["attn"] = None    # each layer's activations are saved tensors of its node(s) now, released with them
        return h, pooled, (hidden if flags[0] else []), (maps if flags[2] else attn)

    @contextlib.contextmanager
    def _node_backward(self, st, grads):
        """Around the backward of one layerwise node: the pass's dropout word bound (its masks regenerated) and unbound on the way
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
        dev = ids.device
        cfg = self.config
        H = _cfg(cfg, "hidden_size")
        heads = _cfg(cfg, "num_attention_heads")
        eps = float(_cfg(cfg, "layer_norm_eps"))
        want_hidden, want_attn = base[:2] if base is not None else (False, False)
        train = self.bert.training if base is not None else self.training
        p_h = float(_cfg(cfg, "hidden_dropout_prob")) if train else 0.0
        p_a = float(_cfg(cfg, "attention_probs_dropout_prob")) if train else 0.0
        seed = self._next_seed()
        nseq, lt = ids.shape
        nvid, T, gh, gw, _ = grid.shape
        L = lt + gh * gw
        M = nseq * L
        bf16, f32 = torch.bfloat16, torch.float32
        n_ex, s2v, starts = repeat

        def new(*shape, dtype=bf16):
            return torch.empty(*shape, dtype=dtype, device=dev)

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
            L = lt + n_keep
            M = nseq * L
        drop_word = self._advance_dropout_stream(dev) if (p_h > 0 or p_a > 0) else None
        ops.dropout_offset_bind(drop_word)
        st = dict(ids=ids, mask=mask, grid=grid, repeat=repeat, seed=seed, p_h=p_h, p_a=p_a, dims=(nseq, nvid, T, gh, gw, lt, L), layers=[],
                  sample=sample, drop_word=drop_word)
        # ---- embeddings: [text ; visual] written straight into one (B', L, 768) buffer ----
        x = new(M, H)
        st["stats_t"] = new(nseq * lt, 2, dtype=f32)
        st["stats_v"] = new(nseq * gh * gw, 2, dtype=f32)
        g_t, b_t, _, _ = self._ln("emb.ln")
        g_v, b_v, _, _ = self._ln("vis.ln")
        word, pos, typ = self._emb("emb.word")[0], self._emb("emb.pos")[0], self._emb("emb.type")[0]
        ops.embed_text_fwd(ids, word, pos, typ, g_t, b_t, x, st["stats_t"], nseq, lt, L, eps, p_h, seed + 1)
        ops.embed_visual_fwd(grid, s2v, n_ex, row_tab, col_tab, self._emb("vis.type")[0], g_v, b_v,
                             x, st["stats_v"], nseq, T, gh, gw, lt, L, eps, p_h, seed + 2)
        cap = self._capture
        if cap is not None:
            cap["embeddings"] = x.view(nseq, L, H).clone()
            cap.update(seed=seed, drop_word=drop_word, stats_t=st["stats_t"], stats_v=st["stats_v"], grid=grid,
                       idx=None if sample is None else sample[0], row_tab=row_tab, col_tab=col_tab)
        # ---- encoder ----
        hidden, attn = [], []
        for i in range(len(self.bert.encoder.layer)):
            ls = seed + 16 * (i + 1)
            if self._inject is not None and i in self._inject:      # test hook: layer-local parity (same input on both sides)
                x = self._inject[i].to(device=dev, dtype=bf16).reshape(M, H).contiguous()
            if want_hidden:
                hidden.append(x.view(nseq, L, H))
            qkv_l, ao_l, in_l, out_l = (self._lin["l%d.%s" % (i, k)] for k in ("qkv", "ao", "inter", "out"))
            g1, b1, _, _ = self._ln("l%d.ln1" % i)
            g2, b2, _, _ = self._ln("l%d.ln2" % i)
            qkv = new(M, 3 * H)
            self._gemm_fwd(x, M, qkv_l, qkv)
            ctx = new(M, H)
            lse = new(nseq, heads, L, dtype=f32) if (need_backward or want_attn) else None
            ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, heads, p_a, ls + 1)
            if want_attn:       # same seed and bound word as the forward: the probabilities its context was made from
                probs = new(nseq, heads, L, L, dtype=f32)
                ops.attention_probs(qkv, mask, lse, probs, nseq, L, lt, heads, p_a, ls + 1)
                attn.append(probs)
            s1 = new(M, H)
            self._gemm_fwd(ctx, M, ao_l, s1, residual=x, res_ld=H, dropout_p=p_h, dropout_seed=ls + 2)
            a = new(M, H)
            st1 = new(M, 2, dtype=f32)
            ops.layernorm_fwd(s1, g1, b1, a, st1, eps)
            u = new(M, in_l.n) if need_backward else None
            gel = new(M, in_l.n)
            if need_backward:
                # u holds gelu'(pre-activation), not the pre-activation: the backward epilogue is then one multiply
                self._gemm_fwd(a, M, in_l, gel, act=ops.ACT_GELU_STASH_GRAD, out2=u, out2_ld=in_l.n)
            else:
                self._gemm_fwd(a, M, in_l, gel, act=ops.ACT_GELU)
            s2 = new(M, H)
            self._gemm_fwd(gel, M, out_l, s2, residual=a, res_ld=H, dropout_p=p_h, dropout_seed=ls + 3)
            y = new(M, H)
            st2 = new(M, 2, dtype=f32)
            ops.layernorm_fwd(s2, g2, b2, y, st2, eps)
            if need_backward:
                st["layers"].append(dict(x=x, qkv=qkv, ctx=ctx, lse=lse, s1=s1, st1=st1, a=a, u=u, gel=gel, s2=s2, st2=st2, seed=ls))
            if cap is not None:
                cap["l%d" % i] = dict(x=x, qkv=qkv, ctx=ctx, lse=lse, s1=s1, st1=st1, a=a, gel=gel, u=u, s2=s2, st2=st2)
            x = y
            if cap is not None:
                cap["layer%d" % i] = x.view(nseq, L, H)
        st["x_last"] = x
        # ---- pooler on the [CLS] rows (row pitch L*768, no gather) ----
        pl = self._lin["pooler"]
        pooled = new(nseq, H)
        self._gemm_fwd(x, nseq, pl, pooled, a_ld=L * H, act=ops.ACT_TANH)
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

    def _dgrad(self, li, dy, rows, out, **kw):
        ops.gemm(mode=ops.CB_GEMM_NN, m=rows, n=li.k, k=li.n, a=dy, a_rows=rows, a_ld=li.n, b=li.w, b_rows=li.n, b_ld=li.k,
                 out=out, out_ld=kw.pop("out_ld", li.k), **kw)

    def _mlp_head_backward(self, st, dlogits, nseq, H):
        """Returns d(pooled) (bf16, [nseq, H])."""
        dev = dlogits.device
        bf16 = torch.bfloat16
        c0, c2, pl = self._lin["cls0"], self._lin["cls2"], self._lin["pooler"]
        dl = torch.empty(nseq, c2.n, dtype=bf16, device=dev)
        ops.pad_cast(dlogits.float().contiguous() if dlogits.dtype != torch.float32 or not dlogits.is_contiguous() else dlogits, dl)
        self._wgrad(c2, dl, st["c1"], nseq)
        ops.colsum(dl, c2.gb, nseq, c2.n)
        dc1 = torch.empty(nseq, c0.n, dtype=bf16, device=dev)
        self._dgrad(c2, dl, nseq, dc1, aux=st["c1"], aux_ld=c0.n, aux_mode=ops.AUX_RELU_MASK)
        self._wgrad(c0, dc1, st["pd"], nseq)
        ops.colsum(dc1, c0.gb, nseq, c0.n)
        dpooled = torch.empty(nseq, H, dtype=bf16, device=dev)
        # d(pooler pre-activation) = (dc1 @ W0) * dropout_mask * tanh'(pooled)
        self._dgrad(c0, dc1, nseq, dpooled, dropout_p=st["p_h"], dropout_seed=st["seed"] + 5, aux=st["pooled"], aux_ld=H,
                    aux_mode=ops.AUX_TANH_GRAD)
        if self._capture is not None:
            self._capture.setdefault("bwd", {}).update(dl=dl, dc1=dc1)
        return dpooled

    def _head_backward(self, st, dout, nseq, H):
        return self._mlp_head_backward(st, dout, nseq, H)

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
            dx = self._layer_backward(st, i, st["layers"][i], dx, sq, cap, None if dattn is None else dattn[i],
                                      None if ret_attn is None else ret_attn[i])
            st["layers"][i] = None     # free this layer's stash
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

    def _layer_backward(self, st, i, ly, dx, sq, cap=None, dattn=None, ret_attn=None, grads=True, split=None):
        """Encoder layer i from the gradient at its output dx ([nseq * L, H] bf16, not written) to the gradient at its input, with
        the layer's stash ly; weight gradients on the side queue sq. dattn: a loss term on the layer's returned attention map,
        ret_attn: the map when retained. grads = False: no parameter gradient is written (a backward that does not accumulate
        into the parameters). split (the backward split at a differentiable map, ClipBertBaseModel.layerwise_autograd): stop at
        the attention and return (d map = dO V^T, hand-over) - the hand-over (dqkv with its V block written, ds1) when split is
        "with_map" (the map's node runs next and finishes the layer in _map_backward), None when it is "map_only"."""
        dev = dx.device
        H = _cfg(self.config, "hidden_size")
        heads = _cfg(self.config, "num_attention_heads")
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        M = nseq * L
        p_h, p_a = st["p_h"], st["p_a"]
        bf16, f32 = torch.bfloat16, torch.float32

        def new(*shape, dtype=bf16):
            return torch.empty(*shape, dtype=dtype, device=dev)

        ls = ly["seed"]
        qkv_l, ao_l, in_l, out_l = (self._lin["l%d.%s" % (i, k)] for k in ("qkv", "ao", "inter", "out"))
        g1, _, dg1, db1 = self._ln("l%d.ln1" % i)
        g2, _, dg2, db2 = self._ln("l%d.ln2" % i)
        dbo, dbao = out_l.gb, ao_l.gb
        if not grads:
            dg1 = db1 = dg2 = db2 = dbo = dbao = None
        # y = LN2(s2), s2 = dropout(gel @ Wo^T + bo) + a
        ds2 = new(M, H)
        ds2d = new(M, H) if p_h > 0 else None
        ops.layernorm_bwd(dx, ly["s2"], ly["st2"], g2, ds2, ds2d, dg2, db2, dbo, p_h, ls + 3)
        dd = ds2d if ds2d is not None else ds2
        gmode = ops.group_wgrad      # the layer's four weight gradients as ONE launch (issued when the last dY, dqkv, exists) or two pairs
        group = gmode in (1, 3, 4)
        pairs = gmode == 4
        wg = [self._wgrad_kw(out_l, dd, ly["gel"], M)]
        if grads and not group:
            sq.run(lambda: ops.gemm(**wg[0]), dd, ly["gel"])
        du = new(M, in_l.n)
        self._dgrad(out_l, dd, M, du, aux=ly["u"], aux_ld=in_l.n, aux_mode=ops.AUX_MUL)
        wg.append(self._wgrad_kw(in_l, du, ly["a"], M))
        if not grads:
            pass
        elif pairs:
            wg_ffn, wg = wg, []
            sq.run(lambda: (ops.gemm_wgrad_group(wg_ffn), ops.colsum(du, in_l.gb, M, in_l.n)), dd, ly["gel"], du, ly["a"])
        elif group:
            sq.run(lambda: ops.colsum(du, in_l.gb, M, in_l.n), du)
        else:
            sq.run(lambda: (ops.gemm(**wg[1]), ops.colsum(du, in_l.gb, M, in_l.n)), du, ly["a"])
        da = new(M, H)
        self._dgrad(in_l, du, M, da, residual=ds2, res_ld=H)
        # a = LN1(s1), s1 = dropout(ctx @ Wao^T + b) + x
        ds1 = new(M, H)
        ds1d = new(M, H) if p_h > 0 else None
        ops.layernorm_bwd(da, ly["s1"], ly["st1"], g1, ds1, ds1d, dg1, db1, dbao, p_h, ls + 2)
        dd1 = ds1d if ds1d is not None else ds1
        wg.append(self._wgrad_kw(ao_l, dd1, ly["ctx"], M))
        if grads and not group:
            sq.run(lambda: ops.gemm(**wg[2]), dd1, ly["ctx"])
        dctx = new(M, H)
        self._dgrad(ao_l, dd1, M, dctx)
        if split is not None:
            if grads and group and wg:           # the weight gradients still pending here; the map's node issues the QKV one
                sq.run(lambda: ops.gemm_wgrad_group(wg), dd, ly["gel"], du, ly["a"], dd1, ly["ctx"])
            dmap = new(nseq, heads, L, L, dtype=f32)
            ops.attention_dprobs(ly["qkv"], dctx, dmap, False, nseq, L, heads)
            if split != "with_map":
                return dmap, None
            dqkv = new(M, 3 * H)
            ops.attention_bwd_dv(ly["qkv"], st["mask"], ly["lse"], dctx, dqkv, nseq, L, lt, heads, p_a, ls + 1)
            return dmap, (dqkv, ds1)
        dqkv = new(M, 3 * H)
        ops.attention_bwd(ly["qkv"], st["mask"], ly["ctx"], dctx, ly["lse"], dqkv, nseq, L, lt, heads, p_a, ls + 1)
        if dattn is not None:      # a loss on attentions[i]: its dQ / dK added into dqkv
            drow = new(nseq, heads, L, dtype=f32)
            if cap is not None:
                cap.setdefault("l%d" % i, {})["dqkv_attn"] = dqkv.clone()
            ops.attention_probs_bwd(ly["qkv"], st["mask"], ly["lse"], dattn, drow, dqkv, nseq, L, lt, heads, p_a, ls + 1)
        if ret_attn is not None:
            _add_retained_attention_grad(ret_attn, ly["qkv"], dctx, nseq, L, heads)
        wg.append(self._wgrad_kw(qkv_l, dqkv, ly["x"], M))
        if not grads:
            pass
        elif group:
            sq.run(lambda: (ops.gemm_wgrad_group(wg), ops.colsum(dqkv, qkv_l.gb, M, 3 * H)), dd, ly["gel"], du, ly["a"], dd1, ly["ctx"], dqkv, ly["x"])
        else:
            sq.run(lambda: (ops.gemm(**wg[3]), ops.colsum(dqkv, qkv_l.gb, M, 3 * H)), dqkv, ly["x"])
        dxn = new(M, H)
        self._dgrad(qkv_l, dqkv, M, dxn, residual=ds1, res_ld=H)
        if cap is not None:
            c = cap.setdefault("l%d" % i, {})
            c.update(dx=dx, ds2=ds2, ds2d=ds2d, du=du, da=da, ds1=ds1, ds1d=ds1d, dctx=dctx, dqkv=dqkv)
            c.setdefault("dxn", dxn)
        return dxn

    def _map_backward(self, st, i, ly, G, handover, sq, grads=True):
        """The rest of encoder layer i's backward from G, the full gradient of its attention map (fp32 [nseq, heads, L, L]), when
        the backward is split at the map: dQ / dK written from G (cb_attention_probs_bwd_store), then the QKV weight gradient and
        the dgrad to the layer input with the residual ds1. handover = (dqkv with its V block, ds1) from _layer_backward, or None
        when the layer's output got no gradient (dV = 0, no residual)."""
        H = _cfg(self.config, "hidden_size")
        heads = _cfg(self.config, "num_attention_heads")
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        M = nseq * L
        dev = G.device
        qkv_l = self._lin["l%d.qkv" % i]
        if handover is None:
            dqkv, ds1 = torch.empty(M, 3 * H, dtype=torch.bfloat16, device=dev), None
            dqkv[:, 2 * H:].zero_()
        else:
            dqkv, ds1 = handover
        drow = torch.empty(nseq, heads, L, dtype=torch.float32, device=dev)
        ops.attention_probs_bwd_store(ly["qkv"], st["mask"], ly["lse"], G, drow, dqkv, nseq, L, lt, heads, st["p_a"], ly["seed"] + 1)
        if grads:
            kw = self._wgrad_kw(qkv_l, dqkv, ly["x"], M)
            sq.run(lambda: (ops.gemm(**kw), ops.colsum(dqkv, qkv_l.gb, M, 3 * H)), dqkv, ly["x"])
        dxn = torch.empty(M, H, dtype=torch.bfloat16, device=dev)
        if ds1 is None:
            self._dgrad(qkv_l, dqkv, M, dxn)
        else:
            self._dgrad(qkv_l, dqkv, M, dxn, residual=ds1, res_ld=H)
        return dxn

    def _embedding_backward(self, st, dx, grid_needs_grad, grads=True):
        """The text and visual embeddings from the gradient at their output dx; returns d visual_inputs (None unless
        grid_needs_grad). grads = False: no parameter gradient is written (the visual kernel's go to scratch)."""
        dev = dx.device
        H = _cfg(self.config, "hidden_size")
        nseq, nvid, T, gh, gw, lt, L = st["dims"]
        p_h = st["p_h"]
        bf16 = torch.bfloat16
        n_ex, s2v, starts = st["repeat"]
        g_t, _, dg_t, db_t = self._ln("emb.ln")
        g_v, _, dg_v, db_v = self._ln("vis.ln")
        (word, dword), (pos, dpos), (typ, dtyp) = self._emb("emb.word"), self._emb("emb.pos"), self._emb("emb.type")
        if grads:
            ops.embed_text_bwd(dx, st["ids"], word, pos, typ, g_t, st["stats_t"], dword, dpos, dtyp, dg_t, db_t, nseq, lt, L, p_h,
                               st["seed"] + 1)
        (row, drow), (col, dcol), (vtyp, dvtyp) = self._emb("vis.row"), self._emb("vis.col"), self._emb("vis.type")
        if not grads:
            if not grid_needs_grad:
                return None
            drow, dcol, dvtyp, dg_v, db_v = (torch.zeros_like(t) for t in (drow, dcol, dvtyp, dg_v, db_v))
        dv_tmp = torch.empty(nseq * gh * gw, H, dtype=torch.float32, device=dev)
        dgrid = torch.empty(nvid, T, gh, gw, H, dtype=bf16, device=dev) if grid_needs_grad else None
        sample = st.get("sample")
        if sample is None:
            ops.embed_visual_bwd(dx, st["grid"], s2v, starts, n_ex, row, col, vtyp, g_v, st["stats_v"], dv_tmp, dgrid, drow, dcol, dvtyp,
                                 dg_v, db_v, nseq, nvid, T, gh, gw, lt, L, p_h, st["seed"] + 2)
        else:
            # sampled visual tokens (see _forward_impl): gradients of the (n_keep x 1) virtual grid, scattered back by index
            idx, gh0, gw0, row_s, col_s = sample
            drow_s, dcol_s = torch.zeros_like(row_s), torch.zeros_like(col_s)
            ops.embed_visual_bwd(dx, st["grid"], s2v, starts, n_ex, row_s, col_s, vtyp, g_v, st["stats_v"], dv_tmp, dgrid, drow_s, dcol_s,
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

    def _head_backward(self, st, douts, nseq, H):
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
            self._wgrad(itm_l, dl, st["pooled"], nseq)
            ops.colsum(dl, itm_l.gb, nseq, itm_l.n)
            self._dgrad(itm_l, dl, nseq, dpre, aux=st["pooled"], aux_ld=H, aux_mode=ops.AUX_TANH_GRAD)
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
            ops.gemm(mode=ops.CB_GEMM_WGRAD, m=vp, n=H, k=R, a=ds, a_rows=R, a_ld=vp, b=st["mlm_t2"], b_rows=R, b_ld=H, out=gword,
                     out_ld=H, out_fp32=1)
            ops.colsum(ds, self._flat.grad[eb["offset"]: eb["offset"] + vp], R, vp)
            dt2 = torch.empty(R, H, dtype=bf16, device=dev)
            ops.gemm(mode=ops.CB_GEMM_NN, m=R, n=H, k=vp, a=ds, a_rows=R, a_ld=vp, b=self._word_bf16, b_rows=vp, b_ld=H, out=dt2, out_ld=H)
            g, _, dg, db = self._ln("mlm_ln")
            dt1 = torch.empty(R, H, dtype=bf16, device=dev)
            ops.layernorm_bwd(dt2, st["mlm_t1"], st["mlm_stats"], g, dt1, None, dg, db, None, 0.0, 0)
            # d(pre-GELU) = dt1 * gelu'(u): a dgrad-style epilogue needs a GEMM, so fold it into the dgrad of transform.dense
            # by first masking dt1 (relu_mask has no gelu form) -> use the NN GEMM of the *identity-free* path below
            du = torch.empty(R, H, dtype=bf16, device=dev)
            _gelu_bwd(dt1, st["mlm_u"], du)
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
