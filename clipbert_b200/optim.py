"""Fused AdamW + gradient clipping over the flat parameter buffers (SURVEY.md §8 f2).

``FusedAdamW`` takes the same arguments as the reference's ``AdamW`` (src/optimization/adamw.py:21-37: param groups
with per-group ``lr`` / ``weight_decay``, ``betas``, ``eps`` = 1e-6, ``correct_bias``) plus the ``ClipBert`` model whose
parameters it owns, so ``setup_e2e_optimizer`` (src/optimization/utils.py:96-130) only swaps the class. One ``step()`` is
two kernel launches (transformer buffer, CNN buffer) instead of ~10 ATen launches per parameter:

    grad-norm clipping (run_video_retrieval.py:477-480)  -> ``clip_grad_norm(max_norm)``: two ``cb_sumsq`` launches; the
                                                            clip coefficient is applied inside the update kernel
    AdamW update (adamw.py:40-103)                        -> ``cb_adamw_step``
    optimizer.zero_grad() (:486)                          -> ``step(zero_grad=True)`` zeroes the gradient in the same pass
    amp O2 master -> model copy (:307-309)                -> the kernel also writes the bf16 tensor-core operands (FrozenBN
                                                            scale folded in), so the next forward does not re-cast weights

``state[p]['exp_avg']`` / ``['exp_avg_sq']`` / ``['step']`` exist with the reference's names (views into two flat fp32
buffers per model half), so ``state_dict()`` / ``load_state_dict()`` and the reference's checkpoint restorer keep working.
"""
import math

import torch
from torch.optim import Optimizer

from . import _lib as L
from . import ops

CHUNK = 65536


def _fn(name, argtypes):
    import ctypes
    f = getattr(L.lib(), name)
    f.argtypes = argtypes
    f.restype = ctypes.c_int
    return f


_cfuncs = {}


def _cfn(name):
    import ctypes
    f = _cfuncs.get(name)
    if f is None:
        vp, i, i64, fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float
        sigs = {"cb_sumsq": [vp, i64, vp, i, vp, vp], "cb_adamw_step": [vp, vp, vp, vp, vp, vp, i, vp, vp, vp, fl, i, vp]}
        f = _cfuncs[name] = _fn(name, sigs[name])
    return f


def _p(t):
    return None if t is None else t.data_ptr()


def sumsq(x, chunks, nchunks, out):
    """cb_sumsq: out[0] += sum of x^2 over the chunk table's elements (include/clipbert_b200.h); cb_sumsq_det under
    torch.use_deterministic_algorithms(True)."""
    if ops.deterministic():
        ops.sumsq_det(x, x.numel(), chunks, nchunks, out, ops._scratch(ops.sumsq_scratch_bytes(x.numel(), chunks, nchunks), x))
        return
    L.check(_cfn("cb_sumsq")(_p(x), x.numel(), _p(chunks), nchunks, _p(out), torch.cuda.current_stream().cuda_stream), "cb_sumsq")


def adamw_step(master, grad, exp_avg, exp_avg_sq, packed, chunks, nchunks, hyper, scales, grad_sumsq, max_norm, zero_grad):
    """cb_adamw_step: clip + AdamW + zero_grad + bf16 operand emission on every element named by the chunk table."""
    L.check(_cfn("cb_adamw_step")(_p(master), _p(grad), _p(exp_avg), _p(exp_avg_sq), _p(packed), _p(chunks), nchunks, _p(hyper), _p(scales),
                                  _p(grad_sumsq), float(max_norm), int(bool(zero_grad)), torch.cuda.current_stream().cuda_stream),
            "cb_adamw_step")


def _require_cuda(dev):
    assert dev.type == "cuda", "FusedAdamW runs on CUDA only (no CPU fallback)"


class FusedAdamW(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True, model=None):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[1]))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(eps))
        if model is None:
            raise ValueError("FusedAdamW needs model=<ClipBert>: it updates the model's flat parameter buffers in place")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias))
        self.model = model
        self._plan = None
        self._pending_max_norm = -1.0
        self._gsq = None
        self.last_grad_norm = None

    # ---- planning: parameters -> chunks of the flat buffers ---------------------------------------------------------
    def _halves(self):
        return [m for m in (self.model.transformer, self.model.cnn) if any(p.requires_grad for p in m.parameters())]

    def _build_plan(self):
        import ctypes
        dev = next(self.model.parameters()).device
        _require_cuda(dev)
        group_of = {}
        for gi, g in enumerate(self.param_groups):
            for p in g["params"]:
                group_of[id(p)] = gi
        halves = []
        for mod in self._halves():
            mod._ensure_ready(dev)
            flat = mod._flat
            segs = {id(s["param"]): s for s in mod.optimizer_segments()}
            rows = []
            views = []
            for e in flat.entries:
                p = e["param"]
                gi = group_of.get(id(p))
                if gi is None or not p.requires_grad:
                    continue
                s = segs.get(id(p), {})
                row_len, soff, emit = int(s.get("row_len", 0)), int(s.get("scale_off", -1)), int(bool(s.get("emit", False)))
                for c0 in range(0, e["numel"], CHUNK):
                    rows.append([e["offset"] + c0, min(CHUNK, e["numel"] - c0), gi, row_len, soff, emit, c0, 0])
                views.append((p, e))
            if not rows:
                continue
            m_buf = torch.zeros_like(flat.master)
            v_buf = torch.zeros_like(flat.master)
            for p, e in views:      # reference state names (adamw.py:62-69), as views of the flat moment buffers
                st = self.state[p]
                old_m, old_v = st.get("exp_avg"), st.get("exp_avg_sq")
                st["exp_avg"], st["exp_avg_sq"] = flat._view(m_buf, e), flat._view(v_buf, e)
                if old_m is not None:      # moments restored by load_state_dict before the first step
                    st["exp_avg"].copy_(old_m)
                    st["exp_avg_sq"].copy_(old_v)
                st.setdefault("step", 0)
            halves.append(dict(mod=mod, flat=flat, chunks=torch.tensor(rows, dtype=torch.int64, device=dev), nchunks=len(rows),
                               exp_avg=m_buf, exp_avg_sq=v_buf, scales=mod.optimizer_scales(), params=[p for p, _ in views]))
            mod._optimizer_emits_packed = True
        ng = len(self.param_groups)
        # per-step hyper-parameters travel through a small RING of pinned staging buffers, each guarded by an event: the host
        # may run several steps ahead of the device (no .item() in the loop), and rewriting ONE pinned buffer before its
        # asynchronous copy has executed would hand step t the learning rate / bias correction of step t+1
        self._hyper_ring = []
        for _ in range(4):
            h = torch.zeros(ng, 8, dtype=torch.float32)
            self._hyper_ring.append([h.pin_memory() if dev.type == "cuda" else h, None])
        self._hyper_slot = 0
        self._hyper_dev = torch.zeros(ng, 8, dtype=torch.float32, device=dev)
        self._gsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self._plan = halves
        # per-group step count (every parameter of a group steps together); restored from a loaded state_dict
        self._group_steps = [max([int(self.state[p].get("step", 0)) for p in g["params"] if p in self.state] or [0])
                             for g in self.param_groups]
        return halves

    def _ensure_plan(self):
        plan = self._plan
        if plan is None or any(not h["flat"].is_current() or h["mod"]._flat is not h["flat"] for h in plan):
            plan = self._build_plan()
        return plan

    # ---- reference loop: clip_grad_norm_(amp.master_params(optimizer), cfg.grad_norm) ----------------------------------
    def clip_grad_norm(self, max_norm):
        """Total gradient norm over every parameter of the optimizer (device tensor, for logging). The clip itself - grads
        scaled by max_norm / (norm + 1e-6) when that is < 1 (torch.nn.utils.clip_grad_norm_) - is folded into the next
        ``step()``; the .grad buffers are left unscaled (they are zeroed by that step)."""
        plan = self._ensure_plan()
        self._gsq.zero_()
        for h in plan:
            sumsq(h["flat"].grad, h["chunks"], h["nchunks"], self._gsq)
        self._pending_max_norm = float(max_norm)
        self.last_grad_norm = self._gsq.sqrt()
        return self.last_grad_norm

    @torch.no_grad()
    def step(self, closure=None, zero_grad=False):
        loss = closure() if closure is not None else None
        plan = self._ensure_plan()
        slot = self._hyper_ring[self._hyper_slot]
        self._hyper_slot = (self._hyper_slot + 1) % len(self._hyper_ring)
        if slot[1] is not None:
            slot[1].synchronize()          # the copy that last read this staging buffer has executed
        hyper_host = slot[0]
        for gi, g in enumerate(self.param_groups):
            self._group_steps[gi] += 1
            t = self._group_steps[gi]
            b1, b2 = g["betas"]
            step_size = g["lr"]
            if g["correct_bias"]:      # adamw.py:81-85
                step_size = step_size * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
            hyper_host[gi] = torch.tensor([g["lr"], step_size, g["weight_decay"], b1, b2, g["eps"], 0.0, 0.0])
        self._hyper_dev.copy_(hyper_host, non_blocking=True)
        if self._hyper_dev.is_cuda:
            slot[1] = torch.cuda.Event()
            slot[1].record()
        clip = self._pending_max_norm > 0
        for h in plan:
            f = h["flat"]
            f.attach_grads()
            adamw_step(f.master, f.grad, h["exp_avg"], h["exp_avg_sq"], f.packed, h["chunks"], h["nchunks"], self._hyper_dev, h["scales"],
                       self._gsq if clip else None, self._pending_max_norm if clip else -1.0, zero_grad)
            for p in h["params"]:
                self.state[p]["step"] += 1
            h["mod"].packed_written_by_optimizer()
        self._pending_max_norm = -1.0
        return loss

    # ---- restoring / re-grouping: the plan (flat moment buffers, per-group step counts) is rebuilt from self.state -------------
    def load_state_dict(self, state_dict):
        """torch's Optimizer.load_state_dict replaces ``self.state[p]`` with fresh tensors. The kernels work on the flat moment
        buffers the plan owns, so the plan is dropped here and rebuilt on the next use: ``_build_plan`` adopts the loaded
        ``exp_avg`` / ``exp_avg_sq`` (copied into the flat buffers, state entries become views again) and the loaded step
        counts - whether the restore happens before the first step (TrainingRestorer, src/utils/load_save.py:245-300) or later."""
        super().load_state_dict(state_dict)
        self._plan = None

    def __setstate__(self, state):
        super().__setstate__(state)
        self._plan = None

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        self._plan = None

    def zero_grad(self, set_to_none=False):
        """Zero the flat gradient buffers (one memset each); ``step(zero_grad=True)`` does it inside the update kernel."""
        for h in self._ensure_plan():
            h["flat"].zero_grad()
