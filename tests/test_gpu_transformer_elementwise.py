"""The transformer half of ClipBERT in training (clipbert_b200/modeling.py): every stage of a forward and a backward, element by
element, against float64 computed from what the stage means, not from the launch descriptors the module builds.

Each stage is fed the run's own bf16 inputs (the module's _capture hooks), so every stage is checked on its own and no drift
builds up over 12 layers, while a wrong row, column, residual, mask seed, bias source, split-K chunk or stale buffer still
shows. Weights are the fp32 nn.Module parameters; the packed bf16 operands are first checked bit-exactly against them rounded
once (the fused QKV operand against cat(query, key, value)).

References and bounds are the kernel tests', not derived again:
  GEMM epilogues and the WGRAD bound        tests/test_gpu_gemm_elementwise.py (reference, w_reference; K-split S <= ceil(P / 64))
  attention ctx / lse / dqkv               tests/test_gpu_attention_elementwise.py (forward_ref, backward_ref)
  LayerNorm, embeddings, colsum, gelu_bwd  tests/test_gpu_memory_bound_kernels.py (_ln_rows, _ln_rows_bwd, their depths)
  dropout multipliers                      tests/dropout_ref.py at the seed and device word the run drew
Pure data movement is bit-exact: pad_cast, the [CLS] scatter of the pooler dgrad (every other row +0), the bf16 adds of the
MLM text-row gradient, the copy of the text rows into the MLM head.

Every parameter gradient is read through p.grad, and the whole flat gradient buffer is accounted for: each element lies in a
checked parameter view or in a padding slot (head rows padded to 8, vocab rows 30522-30527, the MLM bias pad, slot rounding),
and padding stays +0. A parameter the oracle's fp32 autograd gives no gradient on the same batch must have none here either.
ClipBertBaseModel (W6) adds the bf16 adds of the hidden-state gradients (bit-exact, one rounding) and, on the layer whose
attention map carries a loss, cb_attention_probs_bwd's dQ / dK added into dqkv (tests/test_gpu_attention_probs_bwd.py).

Every checked tensor prints "RATIO <stage> <case>-<tensor> <max err / bound>". Backends: "h100" (marked gpu) and "emulator"
(tests/ops_emulator.py replaying the same module on the CPU, for the workloads that fit its budget). CPU fault self-tests plant
faults in real tensors of an emulated step and show that the same check functions reject them, while test_gpu_model's
norm-wise checks would not all notice.
"""
import contextlib
import math
import types

import pytest
import torch

import dropout_ref as D
import ops_emulator as E
import test_gpu_attention_elementwise as A
import test_attention_probs_bwd_emulated as PBE
import test_gpu_attention_probs_bwd as PB
import test_gpu_gemm_elementwise as G
import test_gpu_memory_bound_kernels as MB
from elementwise import BF16, F64, U, _record, check_bf16, check_bitexact, check_bound, check_sum
from util import TOL_GRAD, cosine, make_cfg, relerr

H, HEADS, HD = 768, 12, 64
NL = 12
GELU_FLOOR = {True: MB.GELU_FP32_FLOOR, False: MB.GELU_FP32_FLOOR + MB.GELU_FAST_ERF_FLOOR}     # by emulated


# ------------------------------------------------------------------------------------------------ backends
class Backend:
    def __init__(self, name):
        if name == "h100" and not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        self.emulated = name == "emulator"
        self.dev = torch.device("cpu") if self.emulated else torch.device("cuda:0")

    @contextlib.contextmanager
    def ops(self):
        if self.emulated:       # tests/ops_emulator.py, with cb_attention_probs / _probs_bwd restated for ClipBertBaseModel
            with PBE.emulated_ops():
                yield
        else:
            yield
            torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ workloads
class Work:
    """kind: "retrieval" | "mc" (multiple choice, one score per option) | "pretrain" | "base" (ClipBertBaseModel with hidden
    states and differentiable attentions); counts: repeat count per video."""

    def __init__(self, wid, kind="retrieval", counts=(2, 2), T=2, gh=3, lt=32, p=0.0, frames_grad=False, keep=0, det=False,
                 plan=None, twice=False):
        self.id, self.kind, self.counts, self.T, self.gh, self.lt, self.p = wid, kind, list(counts), T, gh, lt, p
        self.frames_grad, self.keep, self.det, self.plan, self.twice = frames_grad, keep, det, plan, twice

    @property
    def L(self):
        return self.lt + (self.keep or self.gh * self.gh)


WORKS = [
    Work("W1"),
    Work("W2", p=0.1),
    Work("W3", kind="mc", counts=(1, 3, 2), lt=40, p=0.1, frames_grad=True),
    Work("W4", counts=(2,), gh=7, frames_grad=True),
    Work("W5", kind="pretrain", counts=(1, 1), T=1, lt=16, keep=5, p=0.1, frames_grad=True),
    Work("W6", kind="base", counts=(1, 1, 1), p=0.1, frames_grad=True),
    Work("W7", det=True),
    Work("W8-g0", plan=(0, False, 1)),
    Work("W8-g1", plan=(1, False, 1)),
    Work("W8-g4", plan=(4, False, 1)),
    Work("W9", twice=True),
]
EMU_WORKS = ("W1", "W5", "W6")
BASE_HIDDEN = (0, 5)         # W6: hidden states (0 = the embedding output) and the attention map carrying a loss
BASE_ATTN = 7
_SD = {}


def _state_dict(kind):
    from oracle import synth
    if kind not in _SD:
        sd = synth.full_state_dict(42)
        if kind == "pretrain":
            sd = {k: v for k, v in sd.items() if not k.startswith("transformer.classifier.")}
            sd.update({k: v for k, v in synth.transformer_state_dict(60, head="pretraining").items() if k.startswith("transformer.cls.")})
        elif kind in ("mc", "base"):
            sd.update(synth.transformer_state_dict(50, num_labels=1) if kind == "mc" else {})
        _SD[kind] = {k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}
    return _SD[kind]


def _model(be, w):
    """The module whose engine runs the step: the head model, or for "base" the engine of a ClipBertBaseModel (its .bert)."""
    import clipbert_b200 as cb
    if w.kind == "base":
        cfg = make_cfg(hidden_dropout_prob=w.p, attention_probs_dropout_prob=w.p)
        cfg.output_hidden_states = cfg.output_attentions = True
        base = cb.ClipBertBaseModel(cfg)
        res = base.load_state_dict({k[len("bert."):]: v for k, v in _state_dict(w.kind).items() if k.startswith("bert.")})
        assert not res.missing_keys and not res.unexpected_keys
        base.differentiable_attentions = True
        base.to(be.dev).train()
        return base._engine
    cls = {"retrieval": cb.ClipBertForVideoTextRetrieval, "mc": cb.ClipBertForMultipleChoice, "pretrain": cb.ClipBertForPreTraining}[w.kind]
    extra = dict(num_labels=3) if w.kind == "mc" else {}
    if w.keep:
        extra["pixel_random_sampling_size"] = w.keep
    m = cls(make_cfg(hidden_dropout_prob=w.p, attention_probs_dropout_prob=w.p, **extra))
    res = m.load_state_dict(_state_dict(w.kind), strict=False)
    assert set(res.missing_keys) <= {"cls.predictions.decoder.weight", "cls.predictions.decoder.bias"} and not res.unexpected_keys
    return m.to(be.dev).train()


def _batch(w, seed):
    from oracle import synth
    g = torch.Generator().manual_seed(seed)
    nvid, nseq = len(w.counts), sum(w.counts)
    grid = (torch.randn(nvid, w.T, w.gh, w.gh, H, generator=g).abs() * 2).to(BF16)
    ids, mask = synth.synth_text(nseq, w.lt, seed=seed)
    return grid, ids, mask, g


@contextlib.contextmanager
def _knobs(w):
    """torch's deterministic flag and the weight-gradient launch plan (ops.group_wgrad, ops.overlap_wgrad, PDL) of one run."""
    from clipbert_b200 import ops
    prev = torch.are_deterministic_algorithms_enabled(), ops.group_wgrad, ops.overlap_wgrad
    torch.use_deterministic_algorithms(bool(w.det) or prev[0])
    pdl = None
    if w.plan is not None:
        ops.group_wgrad, ops.overlap_wgrad = w.plan[0], w.plan[1]
        pdl = ops.set_pdl(w.plan[2])
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0])
        ops.group_wgrad, ops.overlap_wgrad = prev[1], prev[2]
        if pdl is not None:
            ops.set_pdl(pdl)


def _mlm_grad(scores, labels):
    """d(sum of the per-token CE) / d scores, ignore_index -100, divided by the number of labelled tokens (fp32)."""
    s = scores.detach().double()
    d = torch.softmax(s, -1)
    keep = labels != -100
    d[keep.nonzero(as_tuple=True) + (labels[keep],)] -= 1.0
    d[~keep] = 0.0
    return (d / max(1, int(keep.sum()))).float()


def _step(be, m, w, seed, capture=True):
    """One training forward + backward of random upstream gradients; returns (capture, inputs, upstream gradients, flat grad
    before the backward)."""
    grid, ids, mask, g = _batch(w, seed)
    nseq = ids.shape[0]
    dev = be.dev
    gc = grid.to(dev).requires_grad_(w.frames_grad)
    g0 = None
    with be.ops(), _knobs(w):
        m._capture = {} if capture else None
        try:
            if w.keep:
                import numpy as np
                np.random.seed(seed)                    # get_random_sample_indices draws from numpy's global generator
            if w.kind == "pretrain":
                out = m(ids.to(dev), gc, mask.to(dev), _repeat_counts=w.counts)
                itm, mlm = out["itm_scores"], out["mlm_scores"]
                labels = torch.randint(0, 30522, (nseq, w.lt), generator=g)
                labels[torch.rand(nseq, w.lt, generator=g) < 0.6] = -100
                labels[:, 0] = -100
                up = (torch.randn(nseq, 2, generator=g), _mlm_grad(mlm.cpu(), labels))
                outs = (itm, mlm)
            elif w.kind == "base":
                seq, pooled, hidden, attn = m.bert(ids.to(dev), gc, mask.to(dev))
                L = seq.shape[1]
                up = (torch.randn(nseq, L, H, generator=g).to(BF16), torch.randn(nseq, H, generator=g).to(BF16))
                up += tuple(torch.randn(nseq, L, H, generator=g).to(BF16) for _ in BASE_HIDDEN)
                up += (torch.randn(nseq, HEADS, L, L, generator=g),)
                outs = (seq, pooled) + tuple(hidden[k] for k in BASE_HIDDEN) + (attn[BASE_ATTN],)
            else:
                out = m(ids.to(dev), gc, mask.to(dev), _repeat_counts=w.counts)
                up = (torch.randn(out["logits"].shape, generator=g),)
                outs = (out["logits"],)
            g0 = m._flat.grad.clone() if m._flat.grad is not None else None
            torch.autograd.backward(outs, [u.to(dev) for u in up])
            cap = m._capture
        finally:
            m._capture = None
    return cap, dict(grid=grid, ids=ids, mask=mask, gc=gc, outs=[o.detach() for o in outs]), up, g0


# ------------------------------------------------------------------------------------------------ references
def _gemm(A_, B_, mode, shift=None, res=None, aux=None, aux_mode="none", act="none", out2=False, fp32=False, mult=None):
    """tests/test_gpu_gemm_elementwise.py's reference of one TN (B = [N, K]) or NN (B = [K, N]) launch: ((value, bound),
    (out2 value, bound) or None)."""
    M = A_.shape[0]
    N, K = B_.shape if mode == G.TN else B_.shape[::-1]
    c = types.SimpleNamespace(M=M, N=N, K=K, ntaps=1, mode=mode, tap_w=0, sign=1, scale=False, shift=shift is not None,
                              res=res is not None, act=act, out2=out2, aux=aux_mode, fp32=fp32)
    ins = dict(A=A_, B=B_)
    for k, v in (("shift", shift), ("res", res), ("aux", aux)):
        if v is not None:
            ins[k] = v
    return G.reference(c, ins, mult)


def _wgrad(dy, x, out0):
    """out0 + dy^T x, the WGRAD reference and bound, with the largest K-split the launch may pick."""
    P = dy.shape[0]
    w = types.SimpleNamespace(ntaps=1, K=P, M=dy.shape[1], N=x.shape[1], scale=False, tap_w=0)
    return G.w_reference(w, dict(A=dy, B=x, out0=out0), splits=-(-P // G.BK))


def _colsum(x, pre):
    """cb_colsum: pre + column sums, and the bound of tests/test_gpu_memory_bound_kernels.py::test_colsum."""
    x64 = x.double()
    c = 16 + 8 + math.ceil(x.shape[0] / 128) + 2
    return pre.double() + x64.sum(0), c * U * (pre.double().abs() + x64.abs().sum(0))


def _ln_depth(m):
    blocks = min(math.ceil(m / 4), 264)
    return math.ceil(m / blocks) + 4 + blocks + 8


def _mult(p, seed, word, idx, dev):
    if not p:
        return None
    return torch.from_numpy(D.multipliers(D.effective_seed(seed, word), idx, p)).double().to(dev)


class Checker:
    """Runs the checks of one workload: RATIO lines, the number of checks per stage class, and the gradient views read."""

    def __init__(self, case, be, m, g0):
        self.case, self.be, self.m, self.dev = case, be, m, be.dev
        self.worst, self.count = {}, {}
        self.flat = m._flat
        self.g0 = torch.zeros_like(self.flat.grad) if g0 is None else g0
        self.covered = torch.zeros(self.flat.total, dtype=torch.bool)
        self.params = set()

    def _note(self, kind, what, r):
        _record(kind, "%s-%s" % (self.case, what), r)
        self.worst[kind] = max(self.worst.get(kind, 0.0), r)
        self.count[kind] = self.count.get(kind, 0) + 1

    def bound(self, kind, what, got, ref_bound):
        self._note(kind, what, check_bound("%s %s" % (self.case, what), got, *ref_bound))

    def bf16(self, kind, what, got, ref, **kw):
        self._note(kind, what, check_bf16("%s %s" % (self.case, what), got, ref, **kw))

    def sum(self, kind, what, got, ref, terms, c):
        self._note(kind, what, check_sum("%s %s" % (self.case, what), got, ref, terms, c))

    def exact(self, kind, what, got, ref):
        self._note(kind, what, check_bitexact("%s %s" % (self.case, what), got, ref))

    def _off(self, t):
        return (t.data_ptr() - self.flat.grad.data_ptr()) // 4

    def grad(self, p, rows=None):
        """p.grad (rows: its first `rows` rows) and the value it held before this backward; records the view as checked."""
        assert p.grad is not None and p.grad.data_ptr() >= self.flat.grad.data_ptr()
        off = self._off(p.grad)
        g = p.grad if rows is None else p.grad[:rows]
        n = g.numel()
        if rows is None or rows == p.shape[0]:
            self.params.add(id(p))
        self.covered[off:off + n] = True
        return g, self.g0[off:off + n].view(g.shape)


# ------------------------------------------------------------------------------------------------ the checks
def check_packing(m):
    """The bf16 operands against the fp32 module parameters rounded once; the fp32 bias views equal the parameters."""
    bert = m.bert
    f = m._flat
    ops_ = [("l%d.qkv" % i, [ly.attention.self.query, ly.attention.self.key, ly.attention.self.value]) for i, ly in enumerate(bert.encoder.layer)]
    ops_ += [("l%d.%s" % (i, k), [lin]) for i, ly in enumerate(bert.encoder.layer)
             for k, lin in (("ao", ly.attention.output.dense), ("inter", ly.intermediate.dense), ("out", ly.output.dense))]
    ops_ += [("pooler", [bert.pooler.dense])] + [(k, [lin]) for k, lin in m._head_linears()]
    for key, lins in ops_:
        li = m._lin[key]
        w = torch.cat([l.weight.detach() for l in lins])
        b = torch.cat([l.bias.detach() for l in lins])
        n = w.shape[0]
        check_bitexact("packed " + key, li.w[:n], w.double())
        assert li.w.shape[0] == (n + 7) // 8 * 8 if key in dict(m._head_linears()) else li.w.shape[0] == n, key
        assert bool((li.w[n:].cpu().view(torch.int16) == 0).all()) and bool((li.b[n:].cpu() == 0).all()), key + ": operand padding"
        assert torch.equal(li.b[:n].cpu(), b.cpu()), key + " bias"
    if hasattr(m, "_word_bf16"):
        wt = bert.embeddings.word_embeddings.weight.detach()
        check_bitexact("packed word table", m._word_bf16[:wt.shape[0]], wt.double())
        assert bool((m._word_bf16[wt.shape[0]:].cpu().view(torch.int16) == 0).all()), "word table padding rows"
    assert f.master.data_ptr() == bert.encoder.layer[0].attention.self.query.weight.data_ptr()


def _heads(x, nseq):
    """[nseq * L, k * 768] bf16 -> k float64 CPU tensors [nseq, 12, L, 64]."""
    x = x.detach().cpu().double()
    L = x.shape[0] // nseq
    return [t.reshape(nseq, L, HEADS, HD).permute(0, 2, 1, 3) for t in x.view(nseq, L, -1, H).unbind(2)]


def _merge(t):
    n, h, L, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(n * L, h * d)


class Run:
    """Everything one workload's checks need: the capture, the inputs, the dims and the dropout convention."""

    def __init__(self, be, m, w, cap, inp, up):
        self.be, self.m, self.w, self.cap, self.inp, self.up = be, m, w, cap, inp, up
        self.dev = be.dev
        self.nseq, self.lt = inp["ids"].shape
        self.L = w.L
        self.M = self.nseq * self.L
        self.p = w.p
        self.seed = cap["seed"]
        self.word = None if cap["drop_word"] is None else int(cap["drop_word"].item())
        self.rounded = not be.emulated
        madd = torch.zeros(self.nseq, self.L, dtype=F64)
        madd[:, :self.lt] = (inp["mask"] == 0).double() * -10000.0
        self.madd = madd
        self.eps = float(m.config.layer_norm_eps)
        self.vid = torch.repeat_interleave(torch.arange(len(w.counts)), torch.tensor(w.counts))

    def gmult(self, seed, rows, n):
        return _mult(self.p, seed, self.word, D.gemm_index(rows, n), self.dev)

    def dhidden(self, k):
        """W6: the bf16 gradient of hidden_states[k] the loss hands in, [M, 768] on the device, or None."""
        if self.w.kind != "base" or k not in BASE_HIDDEN:
            return None
        return self.up[2 + BASE_HIDDEN.index(k)].reshape(self.M, H).to(self.dev)

    def dattn(self, i):
        """W6: the fp32 gradient of attentions[i] (float64, CPU), or None."""
        if self.w.kind != "base" or i != BASE_ATTN:
            return None
        return self.up[-1].double()

    def lnmult(self, seed, rows):
        return _mult(self.p, seed, self.word, D.layernorm_index(rows), self.dev)


def check_ln_fwd(ck, tag, x, y, stats, gamma, beta, eps):
    v = x.double()
    yr, mean, rstd, terms = MB._ln_rows(v, gamma.double(), beta.double(), v.abs(), eps)
    ck.bf16("ln", tag, y, yr, k=1, terms=terms, c=32)
    var = ((v - mean[:, None]) ** 2).mean(1)
    ck.sum("ln", tag + ".mean", stats[:, 0], mean, v.abs().mean(1), 32)
    rel = torch.where(var > 0, 1.0 + mean.abs() * rstd, torch.ones_like(var))
    ck.sum("ln", tag + ".rstd", stats[:, 1], rstd, rstd * rel, 32)


def check_ln_bwd(ck, tag, ln, dy, x, stats, dx, dx_drop, mult, dbias=None):
    """dx (and dx_drop = dx * mask), dgamma / dbeta through p.grad, and the fused dense-bias sum of the tensor the dgrad reads."""
    v, d64 = x.double(), dy.double()
    ref, xhat, xt, terms = MB._ln_rows_bwd(d64, v, v.abs(), stats, ln.weight.detach().double())
    ck.bf16("ln", tag + ".dx", dx, ref, k=1, terms=terms, c=32)
    src = dx
    if mult is not None:
        ck.bf16("ln", tag + ".dx_drop", dx_drop, ref * mult, k=1, terms=terms * mult, c=32)
        src = dx_drop
    else:
        assert dx_drop is None
    c = _ln_depth(x.shape[0])
    g, pre = ck.grad(ln.weight)
    ck.sum("bias", tag + ".gamma", g, pre.double() + (d64 * xhat).sum(0), pre.double().abs() + (d64.abs() * xt).sum(0), c + 8)
    g, pre = ck.grad(ln.bias)
    ck.sum("bias", tag + ".beta", g, pre.double() + d64.sum(0), pre.double().abs() + d64.abs().sum(0), c)
    if dbias is not None:
        s64 = src.double()
        g, pre = ck.grad(dbias)
        ck.sum("bias", tag + ".dense_bias", g, pre.double() + s64.sum(0), pre.double().abs() + s64.abs().sum(0), c)


def check_linear_grads(ck, tag, lins, dy, x, with_bias=True):
    """Weight gradients (WGRAD of dy and x, split over the fused pieces) and bias gradients (column sums of dy), via p.grad."""
    o = 0
    for name, lin in lins:
        n = lin.weight.shape[0]
        g, pre = ck.grad(lin.weight)
        ck.bound("wgrad", "%s.%s.w" % (tag, name), g, _wgrad(dy[:, o:o + n], x, pre))
        if with_bias:
            g, pre = ck.grad(lin.bias)
            ck.bound("bias", "%s.%s.b" % (tag, name), g, _colsum(dy[:, o:o + n], pre))
        o += n


def check_layer(ck, r, i, dx_in):
    """Forward and backward of encoder layer i from its captured inputs."""
    m, c, cb = r.m, r.cap["l%d" % i], r.cap["bwd"]["l%d" % i]
    ly = m.bert.encoder.layer[i]
    att = ly.attention
    qkv_l, ao_l, in_l, out_l = (m._lin["l%d.%s" % (i, k)] for k in ("qkv", "ao", "inter", "out"))
    ls = r.seed + 16 * (i + 1)
    M, dev, tag = r.M, r.dev, "l%d" % i
    x = c["x"]
    # ---- forward ----
    ck.bound("fwd", tag + ".qkv", c["qkv"], _gemm(x, qkv_l.w, G.TN, shift=qkv_l.b)[0])
    q, k, v = _heads(c["qkv"], r.nseq)
    ra = (torch.ones(r.nseq, HEADS, r.L, r.L, dtype=F64) if not r.p else
          torch.from_numpy(D.multipliers(D.effective_seed(ls + 1, r.word), D.attention_index(r.nseq, HEADS, r.L), r.p)).double())
    O, bO, lse, blse = A.forward_ref(q, k, v, r.madd, ra, r.rounded)
    ck.bound("attention", tag + ".ctx", c["ctx"], (_merge(O), _merge(bO)))
    ck.bound("attention", tag + ".lse", c["lse"], (lse, blse))
    ck.bound("fwd", tag + ".s1", c["s1"], _gemm(c["ctx"], ao_l.w, G.TN, shift=ao_l.b, res=x, mult=r.gmult(ls + 2, M, H))[0])
    check_ln_fwd(ck, tag + ".ln1", c["s1"], c["a"], c["st1"], att.output.LayerNorm.weight, att.output.LayerNorm.bias, r.eps)
    (gel, o2) = _gemm(c["a"], in_l.w, G.TN, shift=in_l.b, act="stash", out2=True)
    ck.bound("fwd", tag + ".gelu", c["gel"], gel)
    ck.bound("fwd", tag + ".u", c["u"], o2)
    ck.bound("fwd", tag + ".s2", c["s2"], _gemm(c["gel"], out_l.w, G.TN, shift=out_l.b, res=c["a"], mult=r.gmult(ls + 3, M, H))[0])
    y = r.cap["layer%d" % i].reshape(M, H)
    check_ln_fwd(ck, tag + ".ln2", c["s2"], y, c["st2"], ly.output.LayerNorm.weight, ly.output.LayerNorm.bias, r.eps)
    if i + 1 < NL:
        assert r.cap["l%d" % (i + 1)]["x"].data_ptr() == y.data_ptr(), tag + ": the next layer does not read this layer's output"
    # ---- backward ----
    dh = r.dhidden(i + 1)
    if dh is None:
        assert cb["dx"] is dx_in, tag + ": the incoming gradient is not the one the layer above produced"
    else:       # d hidden_states[i + 1] added to the layer above's input gradient: one bf16 add
        ck.exact("adds", tag + ".dx_plus_dhidden", cb["dx"], dx_in.double() + dh.double())
    check_ln_bwd(ck, tag + ".ln2", ly.output.LayerNorm, cb["dx"], c["s2"], c["st2"], cb["ds2"], cb["ds2d"], r.lnmult(ls + 3, M),
                 dbias=ly.output.dense.bias)
    dd = cb["ds2d"] if r.p else cb["ds2"]
    ck.bound("dgrad", tag + ".du", cb["du"], _gemm(dd, out_l.w, G.NN, aux=c["u"], aux_mode="mul")[0])
    ck.bound("dgrad", tag + ".da", cb["da"], _gemm(cb["du"], in_l.w, G.NN, res=cb["ds2"])[0])
    check_ln_bwd(ck, tag + ".ln1", att.output.LayerNorm, cb["da"], c["s1"], c["st1"], cb["ds1"], cb["ds1d"], r.lnmult(ls + 2, M),
                 dbias=att.output.dense.bias)
    dd1 = cb["ds1d"] if r.p else cb["ds1"]
    ck.bound("dgrad", tag + ".dctx", cb["dctx"], _gemm(dd1, ao_l.w, G.NN)[0])
    (do,), (ctx,) = _heads(cb["dctx"], r.nseq), _heads(c["ctx"], r.nseq)
    grads = A.backward_ref(q, k, v, r.madd, ra, ctx, c["lse"], do, r.rounded)
    Gr = r.dattn(i)
    dqkv = (cb["dqkv"] if Gr is None else cb["dqkv_attn"]).view(M, 3, H)
    for j, (name, (ref, b)) in enumerate(zip(("dq", "dk", "dv"), grads)):
        ck.bound("attention", "%s.%s" % (tag, name), dqkv[:, j], (_merge(ref), _merge(b)))
    if Gr is not None:
        # a loss on attentions[i]: cb_attention_probs_bwd adds its dQ / dK into dqkv; dV stays as the context backward left it
        dq0, dk0, _ = _heads(cb["dqkv_attn"], r.nseq)
        fin = cb["dqkv"].view(M, 3, H)
        for j, (name, (ref, b)) in enumerate(zip(("dq", "dk"), PB.probs_bwd_ref(q, k, r.madd, c["lse"], ra, Gr, dq0, dk0, r.rounded))):
            ck.bound("attention", "%s.%s+probs" % (tag, name), fin[:, j], (_merge(ref), _merge(b)))
        ck.exact("attention", tag + ".dv+probs", fin[:, 2], dqkv[:, 2].double())
    ck.bound("dgrad", tag + ".dxn", cb["dxn"], _gemm(cb["dqkv"], qkv_l.w, G.NN, res=cb["ds1"])[0])
    # ---- parameter gradients ----
    check_linear_grads(ck, tag + ".qkv", [("query", att.self.query), ("key", att.self.key), ("value", att.self.value)], cb["dqkv"], x)
    check_linear_grads(ck, tag + ".ao", [("dense", att.output.dense)], dd1, c["ctx"], with_bias=False)
    check_linear_grads(ck, tag + ".inter", [("dense", ly.intermediate.dense)], cb["du"], c["a"])
    check_linear_grads(ck, tag + ".out", [("dense", ly.output.dense)], dd, c["gel"], with_bias=False)
    return cb["dxn"]


def check_embeddings(ck, r):
    """Both halves of the embedding forward and backward (tests/test_gpu_memory_bound_kernels.py's restatements), the frames'
    gradient, and the word table (with the tied MLM decoder's WGRAD in the same slot)."""
    m, cap, dev = r.m, r.cap, r.dev
    emb, vis = m.bert.embeddings, m.bert.visual_embeddings
    nseq, lt, L = r.nseq, r.lt, r.L
    out = cap["embeddings"]
    dx = cap["bwd"]["dx_emb"].view(nseq, L, H)
    ids = r.inp["ids"].to(dev)
    # ---- text ----
    word, pos, typ = emb.word_embeddings.weight.detach(), emb.position_embeddings.weight.detach(), emb.token_type_embeddings.weight.detach()
    w64, p64, t64 = word.double()[ids.reshape(-1)], pos.double()[:lt].repeat(nseq, 1), typ.double()[0]
    v = w64 + p64 + t64
    src = w64.abs() + p64.abs() + t64.abs()
    gam, bet = emb.LayerNorm.weight.detach().double(), emb.LayerNorm.bias.detach().double()
    y, mean, rstd, terms = MB._ln_rows(v, gam, bet, src, r.eps)
    mult = _mult(r.p, r.seed + 1, r.word, D.embedding_index(nseq, L, range(lt)), dev)
    mult = torch.ones_like(y) if mult is None else mult.reshape(nseq * lt, H)
    ck.bf16("embeddings", "text", out[:, :lt].reshape(-1, H), y * mult, k=1, terms=terms * mult, c=32)
    st = cap["stats_t"]
    ck.sum("embeddings", "text.mean", st[:, 0], mean, src.mean(1), 32)
    ck.sum("embeddings", "text.rstd", st[:, 1], rstd, rstd * (1.0 + mean.abs() * rstd), 32)
    dy = dx[:, :lt].reshape(-1, H).double() * mult
    dv, xhat, xt, tdv = MB._ln_rows_bwd(dy, v, src, st, gam)
    P = MB._per_pos(nseq)
    rpb = math.ceil(nseq / P) + 4
    flat = ids.reshape(-1)
    z = lambda n: torch.zeros(n, H, dtype=F64, device=dev)  # noqa: E731
    vocab = word.shape[0]
    cnt = torch.bincount(flat, minlength=vocab).double()[:, None]
    gw_, pre = ck.grad(emb.word_embeddings.weight)
    base, base_b = pre.double(), torch.zeros_like(pre, dtype=F64)
    if r.w.kind == "pretrain" and cap["bwd"].get("ds") is not None:
        # the tied MLM decoder: its WGRAD lands in the same slot first ([vocab_pad, 768]; rows past the vocabulary are padding)
        ds, t2 = cap["bwd"]["ds"], cap["t2"]
        base, base_b = _wgrad(ds[:, :vocab], t2, pre)
    sums, asums, tsums = z(vocab).index_add_(0, flat, dv), z(vocab).index_add_(0, flat, dv.abs()), z(vocab).index_add_(0, flat, tdv)
    ck.sum("embeddings", "word", gw_, base + sums, base_b / U + (cnt + 8) * (base.abs() + asums) + 32 * tsums, 1)
    dpos, apos, tpos = z(pos.shape[0]), z(pos.shape[0]), z(pos.shape[0])
    dpos[:lt], apos[:lt], tpos[:lt] = (t.view(nseq, lt, H).sum(0) for t in (dv, dv.abs(), tdv))
    g, pre = ck.grad(emb.position_embeddings.weight)
    ck._note("embeddings", "pos", MB._check_table("pos", g, pre, dpos, apos, tpos, rpb + P + 8))
    all_depth = rpb + P * lt + 8
    g, pre = ck.grad(emb.token_type_embeddings.weight)
    dt, at, tt = z(2), z(2), z(2)
    dt[0], at[0], tt[0] = dv.sum(0), dv.abs().sum(0), tdv.sum(0)
    ck._note("embeddings", "type", MB._check_table("type", g, pre, dt, at, tt, all_depth))
    g, pre = ck.grad(emb.LayerNorm.weight)
    ck.sum("embeddings", "text.gamma", g, pre.double() + (dy * xhat).sum(0), all_depth * (pre.double().abs() + (dy.abs() * xt).sum(0)), 1)
    g, pre = ck.grad(emb.LayerNorm.bias)
    ck.sum("embeddings", "text.beta", g, pre.double() + dy.sum(0), all_depth * (pre.double().abs() + dy.abs().sum(0)), 1)
    # ---- visual ----
    grid = cap["grid"]                                   # [nvid, T, gh, gw, 768] bf16, after the token sampling
    nvid, T, gh, gw = grid.shape[:4]
    Lv = gh * gw
    assert L == lt + Lv
    row0, col0 = vis.row_position_embeddings.weight.detach(), vis.col_position_embeddings.weight.detach()
    idx = cap["idx"]
    if idx is not None:
        # sampled tokens: a (n_keep x 1) virtual grid whose row table is row[idx // w] + col[idx % w] (fp32), column table 0
        gw0 = r.w.gh
        exact_rows = (row0[idx // gw0].double() + col0[idx % gw0].double())
        ck.exact("embeddings", "sampled.row_table", cap["row_tab"], exact_rows)
        assert bool((cap["col_tab"] == 0).all()) and cap["col_tab"].shape[0] == 1
        g_full = r.inp["grid"].to(dev).view(nvid, T, -1, H)
        ck.exact("embeddings", "sampled.grid", grid.view(nvid, T, -1, H), g_full[:, :, idx].double())
    row, col = cap["row_tab"], cap["col_tab"]
    vid = r.vid.to(dev)
    j = torch.arange(Lv, device=dev)
    g64 = grid.double().view(nvid, T, Lv, H)
    gm, ga = g64.mean(1)[vid].reshape(-1, H), g64.abs().mean(1)[vid].reshape(-1, H)
    r64, c64, vt64 = row.double()[j // gw].repeat(nseq, 1), col.double()[j % gw].repeat(nseq, 1), vis.token_type_embeddings.weight.detach().double()[0]
    vv = gm + r64 + c64 + vt64
    vsrc = ga + r64.abs() + c64.abs() + vt64.abs()
    vgam, vbet = vis.LayerNorm.weight.detach().double(), vis.LayerNorm.bias.detach().double()
    y, mean, rstd, terms = MB._ln_rows(vv, vgam, vbet, vsrc, r.eps)
    mult = _mult(r.p, r.seed + 2, r.word, D.embedding_index(nseq, L, range(lt, L)), dev)
    mult = torch.ones_like(y) if mult is None else mult.reshape(nseq * Lv, H)
    ck.bf16("embeddings", "visual", out[:, lt:].reshape(-1, H), y * mult, k=1, terms=terms * mult, c=32)
    st = cap["stats_v"]
    ck.sum("embeddings", "visual.mean", st[:, 0], mean, vsrc.mean(1), 32)
    ck.sum("embeddings", "visual.rstd", st[:, 1], rstd, rstd * (1.0 + mean.abs() * rstd), 32)
    dy = dx[:, lt:].reshape(-1, H).double() * mult
    dv, xhat, xt, tdv = MB._ln_rows_bwd(dy, vv, vsrc, st, vgam)
    cell = [t.view(nseq, Lv, H).sum(0) for t in (dv, dv.abs(), tdv)]
    if idx is None:
        tables = (("row", vis.row_position_embeddings.weight, j // gw, gw, 0), ("col", vis.col_position_embeddings.weight, j % gw, gh, 0))
    else:       # every kept cell's gradient goes to its row and to its column (torch index_add_ after the kernel)
        gw0 = r.w.gh
        tables = (("row", vis.row_position_embeddings.weight, idx // gw0, 1, gw0), ("col", vis.col_position_embeddings.weight, idx % gw0, 1, gw0))
    for name, p, tidx, per, adds in tables:
        n_tab = p.shape[0]
        sums = [torch.zeros(n_tab, H, dtype=F64, device=dev).index_add_(0, tidx, c_) for c_ in cell]
        g, pre = ck.grad(p)
        ck._note("embeddings", name, MB._check_table(name, g, pre, sums[0], sums[1], sums[2], rpb + P * per + 8 + adds))
    all_depth = rpb + P * Lv + 8
    g, pre = ck.grad(vis.token_type_embeddings.weight)
    ck._note("embeddings", "vtype", MB._check_table("vtype", g, pre, dv.sum(0)[None], dv.abs().sum(0)[None], tdv.sum(0)[None], all_depth))
    g, pre = ck.grad(vis.LayerNorm.weight)
    ck.sum("embeddings", "visual.gamma", g, pre.double() + (dy * xhat).sum(0), all_depth * (pre.double().abs() + (dy.abs() * xt).sum(0)), 1)
    g, pre = ck.grad(vis.LayerNorm.bias)
    ck.sum("embeddings", "visual.beta", g, pre.double() + dy.sum(0), all_depth * (pre.double().abs() + dy.abs().sum(0)), 1)
    dgrid = cap["bwd"]["dgrid"]
    if not r.w.frames_grad:
        assert dgrid is None
        return
    per_vid = [torch.zeros(nvid, Lv, H, dtype=F64, device=dev).index_add_(0, vid, t.view(nseq, Lv, H)) for t in (dv, dv.abs(), tdv)]
    cnt = torch.tensor(r.w.counts, dtype=F64, device=dev)[:, None, None]
    ref = (per_vid[0] / T)[:, None].expand(nvid, T, Lv, H)
    tb = (((cnt + 2) * per_vid[1] + 32 * per_vid[2]) / T)[:, None].expand(nvid, T, Lv, H)
    gh0 = r.w.gh
    full_ref = torch.zeros(nvid, T, gh0 * gh0, H, dtype=F64, device=dev)
    full_tb = torch.zeros_like(full_ref)
    cells = idx if idx is not None else torch.arange(Lv, device=dev)
    full_ref[:, :, cells], full_tb[:, :, cells] = ref, tb
    ck.bf16("embeddings", "dgrid", dgrid.reshape(-1, H), full_ref.reshape(-1, H), k=1, terms=full_tb.reshape(-1, H), c=1)
    assert r.inp["gc"].grad is not None and torch.equal(r.inp["gc"].grad.view(torch.int16), dgrid.view(torch.int16)), "frames' .grad"


def check_pooler(ck, r):
    """pooled from the strided [CLS] rows; the dgrad scattered into the [CLS] rows (every other row +0); its WGRAD and bias."""
    m, cap, nseq, L = r.m, r.cap, r.nseq, r.L
    pl = m._lin["pooler"]
    x_last = cap["layer%d" % (NL - 1)]
    cls_rows = x_last[:, 0]
    ck.bound("heads", "pooled", cap["pooled"], _gemm(cls_rows, pl.w, G.TN, shift=pl.b, act="tanh")[0])
    bw = cap["bwd"]
    dpre = bw["dpre"]
    dxp = bw["dx_pooler"].view(nseq, L, H)
    ck.exact("heads", "dx.non_cls_rows", dxp[:, 1:], torch.zeros(nseq, L - 1, H, dtype=F64))
    ck.bound("dgrad", "pooler", dxp[:, 0], _gemm(dpre, pl.w, G.NN)[0])
    check_linear_grads(ck, "pooler", [("dense", m.bert.pooler.dense)], dpre, cls_rows)
    top = bw["l%d" % (NL - 1)]["dx"].view(nseq, L, H)
    extra = bw["extra"]
    if extra is None:
        assert bw["l%d" % (NL - 1)]["dx"] is bw["dx_pooler"]
    else:       # one bf16 add: the MLM text-row gradient onto the pooler scatter
        ck.exact("heads", "dx.plus_extra", top, dxp.double() + extra.view(nseq, L, H).double())


def check_mlp_head(ck, r):
    m, cap, dev = r.m, r.cap, r.dev
    c0, c2 = m._lin["cls0"], m._lin["cls2"]
    pooled, pd = cap["pooled"], cap["pd"]
    nseq = pooled.shape[0]
    mult = _mult(r.p, r.seed + 5, r.word, D.flat_index(nseq * H).reshape(nseq, H), dev)
    if mult is None:
        assert pd is pooled
    else:
        ref = pooled.double() * mult
        ck.bf16("heads", "pd", pd, ref, k=1, terms=ref, c=1)
    ck.bound("heads", "c1", cap["c1"], _gemm(pd, c0.w, G.TN, shift=c0.b, act="relu")[0])
    ck.bound("heads", "logits", cap["logits"], _gemm(cap["c1"], c2.w, G.TN, shift=c2.b, fp32=True)[0])
    bw = cap["bwd"]
    dlog = r.up[0].double().reshape(nseq, -1).to(dev)
    dl_ref = torch.zeros(nseq, c2.n, dtype=F64, device=dev)
    dl_ref[:, :dlog.shape[1]] = dlog
    ck.exact("heads", "dl", bw["dl"], dl_ref)
    ck.bound("heads", "dc1", bw["dc1"], _gemm(bw["dl"], c2.w, G.NN, aux=cap["c1"], aux_mode="mask")[0])
    ck.bound("heads", "dpre", bw["dpre"], _gemm(bw["dc1"], c0.w, G.NN, aux=pooled, aux_mode="tanh", mult=mult)[0])
    cls = m.classifier
    n2 = cls[2].weight.shape[0]
    check_linear_grads(ck, "cls2", [("linear", cls[2])], bw["dl"][:, :n2], cap["c1"])
    check_linear_grads(ck, "cls0", [("linear", cls[0])], bw["dc1"], pd)


def check_base_outputs(ck, r):
    """ClipBertBaseModel.forward's upstream gradients (_base_output_grads): d pooled through tanh' = 1 - pooled^2 in fp32, rounded
    once to bf16; d sequence_output as the bf16 gradient added onto the pooler scatter (check_pooler)."""
    pooled = r.cap["pooled"].double()
    dp = r.up[1].double().to(r.dev)
    t = 1.0 - pooled * pooled
    ref = dp * t
    ck.bf16("heads", "dpre", r.cap["bwd"]["dpre"], ref, k=1, terms=dp.abs() * (pooled * pooled + t.abs()) + ref.abs(), c=1)
    ck.exact("heads", "dseq", r.cap["bwd"]["extra"], r.up[0].reshape(r.M, H).double())


def check_pretraining_head(ck, r):
    m, cap, dev = r.m, r.cap, r.dev
    nseq, lt, L = r.nseq, r.lt, r.L
    itm_l, t_l = m._lin["itm"], m._lin["mlm_t"]
    pooled = cap["pooled"]
    ck.bound("heads", "itm", cap["itm"], _gemm(pooled, itm_l.w, G.TN, shift=itm_l.b, fp32=True)[0])
    x_last = cap["layer%d" % (NL - 1)]
    ck.exact("heads", "xt", cap["xt"], x_last[:, :lt].reshape(-1, H).double())
    t1, u = _gemm(cap["xt"], t_l.w, G.TN, shift=t_l.b, act="gelu", out2=True)
    ck.bound("heads", "mlm.t1", cap["t1"], t1)
    ck.bound("heads", "mlm.u", cap["mlm_u"], u)
    ln = m.cls.predictions.transform.LayerNorm
    check_ln_fwd(ck, "mlm.ln", cap["t1"], cap["t2"], cap["mlm_stats"], ln.weight, ln.bias, r.eps)
    e = m._spec["mlm_bias"]
    vp = m._word_bf16.shape[0]
    bias = m._flat.master[e["offset"]: e["offset"] + vp]
    ck.bound("heads", "mlm.scores", cap["scores"], _gemm(cap["t2"], m._word_bf16, G.TN, shift=bias, fp32=True)[0])
    bw = cap["bwd"]
    ditm, dscores = (u_.double().to(dev) for u_ in r.up)
    ref = torch.zeros(nseq, itm_l.n, dtype=F64, device=dev)
    ref[:, :2] = ditm
    ck.exact("heads", "itm.dl", bw["dl"], ref)
    ck.bound("heads", "dpre", bw["dpre"], _gemm(bw["dl"], itm_l.w, G.NN, aux=pooled, aux_mode="tanh")[0])
    check_linear_grads(ck, "itm", [("linear", m.cls.seq_relationship)], bw["dl"][:, :2], pooled)
    R = nseq * lt
    v = dscores.shape[-1]
    ref = torch.zeros(R, vp, dtype=F64, device=dev)
    ref[:, :v] = dscores.reshape(R, v)
    ck.exact("heads", "mlm.ds", bw["ds"], ref)
    g, pre = ck.grad(m.cls.predictions.bias)
    ck.bound("bias", "mlm.bias", g, _colsum(bw["ds"][:, :v], pre))
    ck.bound("dgrad", "mlm.dt2", bw["dt2"], _gemm(bw["ds"], m._word_bf16, G.NN)[0])
    check_ln_bwd(ck, "mlm.ln", ln, bw["dt2"], cap["t1"], cap["mlm_stats"], bw["dt1"], None, None)
    dt1 = bw["dt1"].double()
    ck.bf16("heads", "mlm.du", bw["mlm_du"], dt1 * G._gelu_grad(cap["mlm_u"].double()), k=1, a=(dt1.abs() * GELU_FLOOR[r.be.emulated]).cpu())
    ck.bound("dgrad", "mlm.dxt", bw["dxt"], _gemm(bw["mlm_du"], t_l.w, G.NN)[0])
    check_linear_grads(ck, "mlm_t", [("dense", m.cls.predictions.transform.dense)], bw["mlm_du"], cap["xt"])
    full = torch.zeros(nseq, L, H, dtype=F64, device=dev)
    full[:, :lt] = bw["dxt"].view(nseq, lt, H).double()
    ck.exact("heads", "extra", bw["extra"], full.view(-1, H))


def oracle_unused(r):
    """The transformer parameters the oracle's fp32 autograd (oracle.clipbert_ref, the reference restated) gives no gradient, or
    an identically zero one, on the same batch: a loss on every sequence-output element and the pooled output (every head
    reads the encoder only through them)."""
    from oracle import clipbert_ref as R
    sd = {"bert." + n: p.detach().cpu().float().clone().requires_grad_(True) for n, p in r.m.bert.named_parameters()}
    grid = R.repeat_tensor_rows(r.inp["grid"].float(), r.w.counts)
    idx = None if r.cap["idx"] is None else r.cap["idx"].cpu()
    seq, pooled = R.clipbert_base_model(r.inp["ids"], grid, r.inp["mask"], sd, prefix="bert.", sample_indices=idx)
    g = torch.Generator().manual_seed(5)
    ((seq * torch.randn(seq.shape, generator=g)).sum() + (pooled * torch.randn(pooled.shape, generator=g)).sum()).backward()
    return {n for n, t in sd.items() if t.grad is None or not bool((t.grad != 0).any())}


def check_flat(ck, r):
    """Every parameter the oracle trains is checked, every one it leaves without a gradient has none here either (None or
    zero), and every other element of the flat gradient buffer is padding and +0."""
    m = r.m
    unused = oracle_unused(r)
    names = {id(p): n for n, p in m.named_parameters()}
    missing = [names[id(p)] for p in m.parameters() if p.requires_grad and id(p) not in ck.params and names[id(p)] not in unused]
    assert not missing, "%s: parameters whose gradient was not checked: %s" % (ck.case, missing[:8])
    for n, p in m.named_parameters():
        if n in unused and id(p) not in ck.params:
            if p.grad is not None:
                assert not bool((p.grad != 0).any()), "%s: %s has a gradient; the oracle gives it none" % (ck.case, n)
                ck.grad(p)
    rest = ~ck.covered
    bits = m._flat.grad.detach().cpu().view(torch.int32)[rest]
    if bool((bits != 0).any()):
        off = int(rest.nonzero()[int((bits != 0).nonzero()[0])])
        ent = [e["name"] for e in m._flat.entries if e["offset"] <= off < e["offset"] + e["slot"]]
        raise AssertionError("%s: %d padding elements of the flat gradient buffer are not +0; first at %d (slot %s)"
                             % (ck.case, int((bits != 0).sum()), off, ent))


def check_run(r, g0):
    ck = Checker(r.w.id, r.be, r.m, g0)
    check_packing(r.m)
    cap = r.cap
    for key in ("embeddings", "pooled", "bwd", "seed") + tuple("l%d" % i for i in range(NL)):
        assert key in cap, "%s: capture %s missing" % (r.w.id, key)
    if r.w.kind == "pretrain":
        check_pretraining_head(ck, r)
    elif r.w.kind == "base":
        check_base_outputs(ck, r)
    else:
        check_mlp_head(ck, r)
    check_pooler(ck, r)
    dx = cap["bwd"]["l%d" % (NL - 1)]["dx"]
    for i in reversed(range(NL)):
        dx = check_layer(ck, r, i, dx)
    dh = r.dhidden(0)
    if dh is None:
        assert cap["bwd"]["dx_emb"] is dx, "the embeddings' gradient is not layer 0's input gradient"
    else:
        ck.exact("adds", "emb.dx_plus_dhidden", cap["bwd"]["dx_emb"], dx.double() + dh.double())
    check_embeddings(ck, r)
    check_flat(ck, r)
    return ck


def _expected(w):
    """Checked tensors per stage class: 12 layers (5 forward GEMM outputs; ctx, lse, dq, dk, dv; LN1 / LN2 forward with their
    stats and backward, dx_drop with dropout; 4 dgrads; 6 weight gradients; 10 bias / LayerNorm gradients), the pooler, the
    embeddings (text and visual forward, stats and every table; dgrid; the sampled-token tables) and the head; for
    ClipBertBaseModel, the bf16 adds of the hidden-state gradients and the attention-map layer's dQ / dK / dV after
    cb_attention_probs_bwd."""
    drop = 1 if w.p else 0
    e = dict(fwd=5 * NL, attention=5 * NL, ln=(8 + 2 * drop) * NL, dgrad=4 * NL + 1, wgrad=6 * NL + 1, bias=10 * NL + 1)
    e["embeddings"] = 16 + (1 if w.frames_grad else 0) + (2 if w.keep else 0)
    if w.kind == "pretrain":
        e["heads"] = 13
        e["ln"] += 4
        e["dgrad"] += 2
        e["wgrad"] += 2
        e["bias"] += 5
    elif w.kind == "base":
        e["heads"] = 5
        e["attention"] += 3
        e["adds"] = len(BASE_HIDDEN)
    else:
        e["heads"] = 7 + drop
        e["wgrad"] += 2
        e["bias"] += 2
    return e


# ------------------------------------------------------------------------------------------------ the tests
def _params(works, emu):
    return ([pytest.param("h100", w, marks=pytest.mark.gpu, id="h100-" + w.id) for w in works]
            + [pytest.param("emulator", w, id="emulator-" + w.id) for w in works if w.id in emu])


@pytest.mark.parametrize("be_name,w", _params(WORKS, EMU_WORKS))
def test_transformer_training_step_elementwise(be_name, w):
    be = Backend(be_name)
    m = _model(be, w)
    if w.twice:      # a first step whose gradients the second must add to, without zero_grad in between
        _step(be, m, w, seed=101, capture=False)
        assert bool((m._flat.grad != 0).any())
    cap, inp, up, g0 = _step(be, m, w, seed=7)
    r = Run(be, m, w, cap, inp, up)
    ck = check_run(r, g0)
    assert ck.count == _expected(w), "%s: stages checked %s, expected %s" % (w.id, ck.count, _expected(w))


@pytest.mark.parametrize("be_name", [pytest.param("h100", marks=pytest.mark.gpu), "emulator"])
def test_capture_changes_nothing(be_name):
    """A training step with _capture set and one without, under torch.use_deterministic_algorithms(True): the same bits in
    the outputs and every gradient, and on the device the same number of launches."""
    from clipbert_b200 import ops
    be = Backend(be_name)
    w = Work("W2-capture", p=0.1, counts=(1, 2), lt=16, det=True)
    res = []
    for capture in (True, False):
        m = _model(be, w)
        n0 = ops.launch_count() if not be.emulated else 0
        cap, inp, up, _ = _step(be, m, w, seed=3, capture=capture)
        n = ops.launch_count() - n0 if not be.emulated else 0
        res.append((m._flat.grad.detach().cpu().clone(), n, inp["outs"][0].cpu()))
    assert torch.equal(res[0][2].view(torch.int32), res[1][2].view(torch.int32)), "logits differ with the capture on"
    assert torch.equal(res[0][0].view(torch.int32), res[1][0].view(torch.int32)), "gradients differ with the capture on"
    assert res[0][1] == res[1][1], "launch counts differ: %d with the capture, %d without" % (res[0][1], res[1][1])


# ------------------------------------------------------------------------------------------------ CPU fault self-tests
# Each fault is planted in a real emulated W1 step (a p.grad or a captured tensor replaced by the faulty value) and must be
# rejected by the same check function the workload tests run; the unfaulted run passes it first.
@pytest.fixture(scope="module")
def emu_w1():
    be = Backend("emulator")
    w = WORKS[0]
    m = _model(be, w)
    cap, inp, up, g0 = _step(be, m, w, seed=7)
    return Run(be, m, w, cap, inp, up)


@contextlib.contextmanager
def _planted(p, value):
    """p.grad holds `value` inside the block, its own value again afterwards."""
    saved = p.grad.clone()
    p.grad.copy_(value)
    try:
        yield
    finally:
        p.grad.copy_(saved)


def _rejected(what, check, p=None, value=None, good=None):
    """check() passes as the run left it and fails with the fault planted (p.grad = value, or check applied to the faulted
    run); prints the relerr and cosine test_gpu_model's norm-wise comparison would see."""
    check()
    if p is not None:
        good = p.grad.clone()
        e, c = relerr(value, good), cosine(value, good)
        ctx = _planted(p, value)
    else:
        e, c = relerr(value, good), cosine(value, good)
        ctx = contextlib.nullcontext()
    print("FAULT %s relerr %.3g cosine %.6f (norm-wise acceptance, relerr < %g with cosine > 0.999: %s)"
          % (what, e, c, TOL_GRAD, e < TOL_GRAD and c > 0.999))
    with ctx, pytest.raises(AssertionError, match="out of bound|not bit-exact"):
        check()
    return e, c


def _layer(r, i):
    return r.m.bert.encoder.layer[i], r.cap["l%d" % i], r.cap["bwd"]["l%d" % i]


def _ck(r):
    return Checker("fault", r.be, r.m, None)


def test_fault_key_bias_gradient_zero_is_rejected_but_passes_the_normwise_check(emu_w1):
    """One layer's key.bias gradient left at zero: rejected by check_linear_grads; test_gpu_model's check of key.bias (norm below
    0.05 of the query bias gradient's) accepts it."""
    r = emu_w1
    ly, c, cb = _layer(r, 5)
    att = ly.attention.self
    lins = [("query", att.query), ("key", att.key), ("value", att.value)]
    bad = torch.zeros_like(att.key.bias.grad)
    assert float(bad.norm()) < 0.05 * float(att.query.bias.grad.norm())
    _rejected("key.bias=0", lambda: check_linear_grads(_ck(r), "l5.qkv", lins, cb["dqkv"], c["x"]), att.key.bias, bad)


def test_fault_ln2_gamma_missing_the_last_row_is_rejected_but_passes_the_normwise_check(emu_w1):
    r = emu_w1
    i = 3
    ly, c, cb = _layer(r, i)
    ln = ly.output.LayerNorm
    d64, v = cb["dx"].double(), c["s2"].double()
    _, xhat, _, _ = MB._ln_rows_bwd(d64, v, v.abs(), c["st2"], ln.weight.detach().double())
    bad = (d64[:-1] * xhat[:-1]).sum(0).float()
    e, cs = _rejected("ln2.gamma-last-row", lambda: check_ln_bwd(_ck(r), "l3.ln2", ln, cb["dx"], c["s2"], c["st2"], cb["ds2"], cb["ds2d"],
                                                                 r.lnmult(r.seed + 16 * (i + 1) + 3, r.M), dbias=ly.output.dense.bias),
                      ln.weight, bad)
    assert e < TOL_GRAD and cs > 0.999


def test_fault_ffn_out_wgrad_missing_its_last_k_chunk_is_rejected(emu_w1):
    r = emu_w1
    ly, c, cb = _layer(r, 7)
    last = (r.M - 1) // G.BK * G.BK
    bad = (cb["ds2"][:last].double().t() @ c["gel"][:last].double()).float()
    _rejected("out.w-last-k-chunk", lambda: check_linear_grads(_ck(r), "l7.out", [("dense", ly.output.dense)], cb["ds2"], c["gel"], with_bias=False),
              ly.output.dense.weight, bad)


def test_fault_pooler_dgrad_written_to_row_1_is_rejected(emu_w1):
    """The last sequence's [CLS] gradient written to its row 1 instead of row 0: rejected by check_pooler."""
    import copy
    r = emu_w1
    good = r.cap["bwd"]["dx_pooler"]
    bad = good.view(r.nseq, r.L, H).clone()
    bad[-1, 1], bad[-1, 0] = bad[-1, 0], 0
    rb = copy.copy(r)
    rb.cap = dict(r.cap, bwd=dict(r.cap["bwd"], dx_pooler=bad.view(-1, H)))
    check_pooler(_ck(r), r)
    e, c = relerr(bad, good.view(bad.shape)), cosine(bad, good.view(bad.shape))
    print("FAULT pooler-row-1 relerr %.3g cosine %.6f" % (e, c))
    with pytest.raises(AssertionError, match="not bit-exact"):
        check_pooler(_ck(rb), rb)


def test_fault_visual_gradient_missing_one_repeat_is_rejected(emu_w1):
    """The visual row-table gradient without the last sequence (one repeat of a video repeated twice), as the emulated
    cb_embed_visual_bwd gives it from the step's own tensors with that sequence's rows left out: rejected by check_embeddings."""
    r = emu_w1
    m, cap = r.m, r.cap
    vis = m.bert.visual_embeddings
    nseq, lt, L, gh = r.nseq, r.lt, r.L, r.w.gh
    dh = cap["bwd"]["dx_emb"].clone().view(nseq, L, H)
    dh[-1] = 0
    g_v = vis.LayerNorm.weight.detach()
    drow = torch.zeros_like(vis.row_position_embeddings.weight)
    z = lambda t: torch.zeros_like(t)  # noqa: E731
    E.embed_visual_bwd(dh.view(-1, H), cap["grid"], None, None, r.w.counts[0], cap["row_tab"], cap["col_tab"],
                       vis.token_type_embeddings.weight.detach(), g_v, cap["stats_v"], torch.zeros(nseq * gh * gh, H), None, drow,
                       z(vis.col_position_embeddings.weight), z(vis.token_type_embeddings.weight), z(g_v), z(g_v),
                       nseq, len(r.w.counts), r.w.T, gh, gh, lt, L, 0.0, 0)
    _rejected("visual-row-one-repeat-missing", lambda: check_embeddings(_ck(r), r), vis.row_position_embeddings.weight, drow)


def test_fault_ffn_in_bias_before_the_gelu_derivative_is_rejected(emu_w1):
    """intermediate.dense.bias summed from d gelu (the dgrad before the multiply by gelu'(u)) instead of du."""
    r = emu_w1
    ly, c, cb = _layer(r, 9)
    out_l = r.m._lin["l9.out"]
    bad = (cb["ds2"].double() @ out_l.w.double()).to(BF16).double().sum(0).float()
    _rejected("inter.b-before-gelu'", lambda: check_linear_grads(_ck(r), "l9.inter", [("dense", ly.intermediate.dense)], cb["du"], c["a"]),
              ly.intermediate.dense.bias, bad)
