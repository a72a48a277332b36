"""ClipBert: CNN + transformer, the module the reference task scripts instantiate
(``src/modeling/e2e_model.py:13-50``). Same constructor, same ``forward(batch: dict) -> dict``,
same attribute names (``.cnn``, ``.transformer``, ``.retrieval``), so ``src/tasks/run_*.py`` can
use it unchanged; parameter names still contain "cnn" / "grid_encoder" / "transformer" so that
``setup_e2e_optimizer`` (src/optimization/utils.py:96-161) yields its 8 parameter groups.
"""
import contextlib

import torch
import torch.distributed as dist
from torch import nn

from .grid_feat import GridFeatBackbone
from .modeling import (ClipBertForMultipleChoice, ClipBertForPreTraining, ClipBertForRegression,  # noqa: F401
                       ClipBertForSequenceClassification, ClipBertForVideoTextRetrieval)


def allreduce_flat(grads, group=None, average=True, async_op=False):
    """Sum (or average) a list of flat gradient buffers over the data-parallel group, in place.

    The H100 replacement of ``hvd.DistributedOptimizer``'s per-parameter allreduce + ``synchronize()``
    (src/tasks/run_video_retrieval.py:299-301,432): two flat fp32 buffers, one NCCL all-reduce each.
    """
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return []
    ws = dist.get_world_size(group)
    nccl = dist.get_backend(group) == "nccl"
    works = []
    for g in grads:
        if average and nccl:
            works.append(dist.all_reduce(g, op=dist.ReduceOp.AVG, group=group, async_op=async_op))   # one pass, 1/N inside NCCL
        else:
            if average:
                g.mul_(1.0 / ws)
            works.append(dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group, async_op=async_op))
    return works


class _Bf16WireWork:
    """One slice of a gradient buffer on its way through the bf16 wire format: ``wait()`` makes the caller's stream wait for the
    all-reduce and for the cast of the averaged values back into the fp32 buffer (both enqueued on the exchange's side stream)."""

    def __init__(self, event):
        self.event = event

    def wait(self):
        torch.cuda.current_stream().wait_event(self.event)


class _StreamWork:
    """``Work.wait()`` for an exchange enqueued on a side stream: the caller's stream waits for its end."""

    def __init__(self, event):
        self.event = event

    def wait(self):
        torch.cuda.current_stream().wait_event(self.event)


class _ClipLseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels):
        from . import ops
        z = logits.detach()
        z = (z if z.dtype == torch.float32 else z.float()).contiguous()
        n_clips, nseq, ncls = z.shape
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
        dz = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        ops.clip_lse_loss(z, labels.to(torch.int64).contiguous(), loss, dz, n_clips, nseq, ncls, 1.0)
        ctx.dz, ctx.in_dtype = dz, logits.dtype
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        dz, ctx.dz = ctx.dz, None
        return (dz * g).to(ctx.in_dtype), None


class _ClipPoolCeLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, pool):
        from . import ops
        z = logits.detach()
        z = (z if z.dtype == torch.float32 else z.float()).contiguous()
        n_clips, nseq, ncls = z.shape
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
        dz = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        ops.clip_pool_ce_loss(z, labels.to(torch.int64).contiguous(), loss, dz, n_clips, nseq, ncls, pool, 1.0)
        ctx.dz, ctx.in_dtype = dz, logits.dtype
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        dz, ctx.dz = ctx.dz, None
        return (dz * g).to(ctx.in_dtype), None, None


def clip_pool_loss(logits, labels, pool_method="lse"):
    """Clip aggregation + cross-entropy loss of the training loops for every ``score_agg_func`` of the reference
    (src/tasks/run_video_retrieval.py:404-422, run_video_qa.py:484-501): "lse" (the shipped configs), "mean", "max" - one fused
    forward+backward kernel each. ``logits``: ``(n_clips, B', C)`` (``torch.stack`` of the per-clip logits, what
    ``ClipBert.forward_clips`` returns); ``labels``: ``(B',)`` int64; returns the scalar mean loss with autograd support."""
    if isinstance(logits, (list, tuple)):
        logits = torch.stack(list(logits))
    if pool_method == "lse":
        return _ClipLseLoss.apply(logits, labels)
    if pool_method not in ("mean", "max"):
        raise ValueError("Invalid value for pool_method, got %s, expect one of [`mean`, `max`, `lse`]" % pool_method)
    return _ClipPoolCeLoss.apply(logits, labels, 1 if pool_method == "mean" else 2)


def clip_lse_loss(logits, labels):
    """Clip aggregation + loss of the training loops with ``pool_method == "lse"``
    (src/tasks/run_video_retrieval.py:404-422, run_video_qa.py:484-501) as one fused forward+backward kernel.

    ``logits``: the ``(n_clips, B', C)`` tensor the reference builds with ``torch.stack(logits)`` (what
    ``ClipBert.forward_clips`` returns); ``labels``: ``(B',)`` int64. Returns the scalar
    ``mean_b(logsumexp_{k,c} z[k,b,c] - logsumexp_k z[k,b,y_b])`` with autograd support."""
    if isinstance(logits, (list, tuple)):
        logits = torch.stack(list(logits))
    return _ClipLseLoss.apply(logits, labels)


class ClipBert(nn.Module):
    def __init__(self, config, input_format="BGR", detectron2_model_cfg=None, transformer_cls=ClipBertForVideoTextRetrieval,
                 freeze_at=2):
        super().__init__()
        self.config = config
        self.detectron2_model_cfg = detectron2_model_cfg
        self.cnn = GridFeatBackbone(detectron2_model_cfg=detectron2_model_cfg, config=config, input_format=input_format,
                                    freeze_at=freeze_at)
        self.transformer = transformer_cls(config)
        self.retrieval = transformer_cls == ClipBertForVideoTextRetrieval

    def forward(self, batch):
        # used to make visual feature copies (repeat_tensor_rows is fused into the visual-embedding kernel)
        repeat_counts = batch["n_examples_list"]
        del batch["n_examples_list"]
        visual_features = self.cnn(batch["visual_inputs"])
        batch["visual_inputs"] = visual_features
        if self.retrieval:
            batch["sample_size"] = len(repeat_counts)  # batch size
        zeroed = self._zero_grads_beside_the_transformer_forward(visual_features)
        out = self.transformer(_repeat_counts=list(repeat_counts), **batch)
        if zeroed is not None:
            torch.cuda.current_stream().wait_event(zeroed)      # before the first weight gradient of the backward is written
        return out

    # ``optimizer.zero_grad()`` of the reference loop (run_video_retrieval.py:486) as part of the step itself: with
    # ``model.zero_grad_in_forward = True`` the two flat gradient buffers (595 MB) are cleared on a side stream while the
    # transformer forward runs - its GEMMs are latency-bound and leave HBM idle - instead of by a serial fill before the step.
    # For loops that call forward exactly once per optimizer step (every reference task at gradient_accumulation_steps 1);
    # leave it off when accumulating gradients over several forward/backward passes (``no_sync``), and with FusedAdamW's
    # ``step(zero_grad=True)``, which already clears the buffer in the optimizer's own pass.
    zero_grad_in_forward = False

    def _zero_grads_beside_the_transformer_forward(self, like):
        if not (self.zero_grad_in_forward and self.training and torch.is_grad_enabled()):
            return None
        grads = self.flat_grads()
        if not grads:
            return None
        if not like.is_cuda:                 # (host-logic tests on emulated ops: no streams)
            for g in grads:
                g.zero_()
            return None
        side = getattr(self, "_zero_stream", None)
        if side is None:
            side = self._zero_stream = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())           # after the previous step's exchange / optimizer read them
        with torch.cuda.stream(side):
            for g in grads:
                g.zero_()
            ev = torch.cuda.Event()
            ev.record(side)
        return ev

    def encode_clips(self, visual_inputs, num_clips):
        """CNN half only: ``(B, num_clips * num_frm, 3, H, W)`` frames -> the grid features of the ``B * num_clips``
        (video, clip) units, ``(B * num_clips, num_frm, h, w, 768)``, to be handed to ``forward_clips(..., grid=...)``.

        The reference's ``inference_retrieval`` re-runs the CNN on the same clip for every caption mini-batch of a video
        (1000 captions / eval_bsz times, src/tasks/run_video_retrieval.py:639-666); computing the grid once per video is
        the same arithmetic (SURVEY.md §8 f1)."""
        bsz, frames = visual_inputs.shape[0], visual_inputs.shape[1]
        assert frames % num_clips == 0, "visual_inputs must hold num_clips * num_frm frames per video"
        return self.cnn(visual_inputs.reshape((bsz * num_clips, frames // num_clips) + tuple(visual_inputs.shape[2:])))

    def forward_clips(self, batch, num_clips, grid=None):
        """All ``num_clips`` clips of a step in ONE pass (SURVEY.md §8 f1, "clip batching").

        The reference loops ``for clip_idx in range(num_clips): model(mini_batch)`` over
        ``visual_inputs.view(B, num_clips, num_frm, ...)[:, clip_idx]`` and stacks the logits
        (src/tasks/run_video_retrieval.py:388-404, run_video_qa.py:470-486). Nothing on the path mixes rows of
        different (video, clip) units (FrozenBN, per-sequence attention, per-row LayerNorm), so running the
        ``B * num_clips`` units as one batch is the same arithmetic with twice/four times the GEMM rows and
        1/num_clips of the launches. ``batch`` is the reference batch dict with ``visual_inputs`` still
        ``(B, num_clips * num_frm, 3, H, W)``; returns ``dict(logits=(num_clips, B', C))`` - the tensor the
        reference builds with ``torch.stack(logits)`` - for the caller's clip aggregation + loss. Only the
        dropout streams differ from the loop (one seed per pass instead of one per clip).

        ``grid``: features from ``encode_clips`` of the same videos; the CNN is then skipped and ``batch`` needs no
        ``visual_inputs`` (caption mini-batches of one video at inference).
        """
        counts = [int(c) for c in batch["n_examples_list"]]
        if grid is not None:
            assert grid.shape[0] == len(counts) * num_clips, "grid must come from encode_clips of the same videos"
            vis, bsz = None, len(counts)
            dev = grid.device
        else:
            vis = batch["visual_inputs"]
            bsz, frames = vis.shape[0], vis.shape[1]
            assert frames % num_clips == 0, "visual_inputs must hold num_clips * num_frm frames per video"
            dev = vis.device
        key = (tuple(counts), num_clips, str(dev))
        plan = getattr(self, "_clip_plan", None)
        if plan is None or plan[0] != key:
            # text rows of unit (b, c) = the rows of video b; output row (c, b, e) <- pass row (b, c, e)
            starts = [0]
            for c in counts:
                starts.append(starts[-1] + c)
            gather = [starts[b] + e for b in range(bsz) for _c in range(num_clips) for e in range(counts[b])]
            unit0 = [num_clips * starts[b] for b in range(bsz)]
            scatter = [unit0[b] + c * counts[b] + e for c in range(num_clips) for b in range(bsz) for e in range(counts[b])]
            plan = (key, torch.tensor(gather, dtype=torch.int64, device=dev), torch.tensor(scatter, dtype=torch.int64, device=dev),
                    [counts[b] for b in range(bsz) for _c in range(num_clips)])
            self._clip_plan = plan
        _, gather, scatter, unit_counts = plan
        mb = dict(text_input_ids=batch["text_input_ids"].index_select(0, gather),
                  text_input_mask=batch["text_input_mask"].index_select(0, gather), labels=None)
        if grid is None:
            mb.update(visual_inputs=vis.reshape((bsz * num_clips, frames // num_clips) + tuple(vis.shape[2:])), n_examples_list=unit_counts)
            logits = self.forward(mb)["logits"]
        else:
            if self.retrieval:
                mb["sample_size"] = len(unit_counts)
            logits = self.transformer(visual_inputs=grid, _repeat_counts=list(unit_counts), **mb)["logits"]
        if logits.shape[0] == scatter.shape[0]:
            return dict(logits=logits.index_select(0, scatter).view(num_clips, -1, logits.shape[-1]))
        # multiple choice: calc_loss already folded the options of a unit into one row (modeling.py:436-437)
        assert logits.shape[0] == bsz * num_clips
        return dict(logits=logits.view(bsz, num_clips, -1).permute(1, 0, 2).contiguous())

    def load_separate_ckpt(self, cnn_weights_path=None, bert_weights_path=None):
        if cnn_weights_path:
            self.cnn.load_state_dict(cnn_weights_path)
        if bert_weights_path:
            sd = torch.load(bert_weights_path, map_location="cpu") if isinstance(bert_weights_path, str) else bert_weights_path
            own = self.transformer.state_dict()
            self.transformer.load_state_dict({k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}, strict=False)
            self.transformer.mark_weights_updated()

    def freeze_cnn_backbone(self):
        for n, p in self.cnn.feature.named_parameters():
            p.requires_grad = False

    # keys the reference checkpoints carry for parts of detectron2 that are dead on this path (SURVEY.md App. B): never an error
    _DEAD_D2_KEYS = ("cnn.feature.proposal_generator.", "cnn.feature.roi_heads.", "cnn.feature.pixel_mean", "cnn.feature.pixel_std")

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Accepts the reference checkpoint layout. The dead d2 heads and BatchNorm's ``num_batches_tracked`` are dropped
        silently; with ``strict=True`` (the default, as ``model.load_state_dict(ckpt)`` in the reference's TrainingRestorer,
        src/utils/load_save.py:283-300) any OTHER unexpected key and any missing key raises, like ``nn.Module.load_state_dict``."""
        own = self.state_dict()
        dead = [k for k in state_dict if k.startswith(self._DEAD_D2_KEYS) or k.endswith("num_batches_tracked")]
        sd = {k: v for k, v in state_dict.items() if k in own}
        if strict:
            unexpected = sorted(k for k in state_dict if k not in own and k not in dead)
            missing = sorted(k for k in own if k not in state_dict)
            if unexpected or missing:
                raise RuntimeError("Error(s) in loading state_dict for ClipBert: missing keys %s, unexpected keys %s" % (missing[:8], unexpected[:8]))
        out = super().load_state_dict(sd, strict=False)
        self.cnn.mark_weights_updated()
        self.transformer.mark_weights_updated()
        return out

    # ---- data-parallel gradient exchange (replaces hvd.DistributedOptimizer.synchronize) -----------
    def flat_grads(self):
        out = []
        for m in (self.transformer, self.cnn):
            if m._flat is not None and m._flat.grad is not None:
                out.append(m._flat.grad)
        return out

    def zero_grad(self, set_to_none=False):
        for m in (self.transformer, self.cnn):
            if m._flat is not None and m._flat.grad is not None:
                m._flat.grad.zero_()

    # ---- NVLS exchange: this library's own all-reduce through the NVSwitch (csrc/nvls.cu) -------------------------------
    def _nvls_exchange(self, tensors, ctas=None):
        """All-reduce slices of the symmetric-memory gradient buffers on the communication stream. Each slice: cross-rank
        barrier (every rank has finished writing it - stream order on each rank), cb_nvls_allreduce_f32, barrier (every
        rank's 1/world slice has been stored everywhere)."""
        from . import ops
        import torch.distributed._symmetric_memory as symm
        dp = self._dp
        group = dp["group"] if dp["group"] is not None else dist.group.WORLD
        world = dist.get_world_size(group)
        comm = dp.get("comm_stream")
        if comm is None:
            comm = dp["comm_stream"] = torch.cuda.Stream()
        comm.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(comm):
            for t in tensors:
                key = t.untyped_storage().data_ptr()
                hdl = dp["handles"].get(key)
                if hdl is None:                      # first use (an eager warm-up step, never under graph capture): collective
                    owner = next(m._flat.grad for m in (self.transformer, self.cnn)
                                 if m._flat is not None and m._flat.grad.untyped_storage().data_ptr() == key)
                    hdl = dp["handles"][key] = symm.rendezvous(owner, group)
                    if not hdl.multicast_ptr:
                        raise RuntimeError("NVLS exchange: this system exposes no multicast mapping (use exchange='nccl')")
                hdl.barrier(channel=0)
                ops.nvls_allreduce(hdl.multicast_ptr + 4 * t.storage_offset(), t.numel(), hdl.rank, world,
                                   1.0 / world if dp["average"] else 1.0, dp["max_ctas"] if ctas is None else ctas)
                hdl.barrier(channel=0)
            ev = torch.cuda.Event()
            ev.record(comm)
        return [_StreamWork(ev)]

    def _bf16_wire_exchange(self, tensors):
        """The all-reduce in the reference's wire precision: amp O2 keeps fp16 gradients and Horovod all-reduces them as they
        are (src/tasks/run_video_retrieval.py:299-309,432) - 2 bytes per parameter, the 297 MB of SURVEY.md §8d - whereas the flat
        buffers here accumulate in fp32. Each slice is cast into a persistent bf16 shadow of its buffer (cb_cast_scale), averaged
        over the ranks in bf16, and cast back (cb_cast_bf16_f32), all on one side stream so that neither cast nor collective
        sits on the backward's critical path. Halves the NVLink payload and the time NCCL's CTAs share the SMs with the backward."""
        from . import ops
        dp = self._dp
        group = dp["group"]
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return []
        ws = dist.get_world_size(group)
        nccl = dist.get_backend(group) == "nccl"
        comm = dp.get("wire_stream")
        if comm is None:
            comm = dp["wire_stream"] = torch.cuda.Stream()
        comm.wait_stream(torch.cuda.current_stream())          # the gradients of these slices are complete in stream order
        with torch.cuda.stream(comm):
            for t in tensors:
                key = t.untyped_storage().data_ptr()
                shadow = dp["shadows"].get(key)
                if shadow is None:
                    owner = next(m._flat.grad for m in (self.transformer, self.cnn)
                                 if m._flat is not None and m._flat.grad is not None and m._flat.grad.untyped_storage().data_ptr() == key)
                    shadow = dp["shadows"][key] = torch.empty(owner.numel(), dtype=torch.bfloat16, device=owner.device)
                lo = t.storage_offset()
                s = shadow[lo: lo + t.numel()]
                ops.cast_scale(t, s)
                if dp["average"] and nccl:
                    dist.all_reduce(s, op=dist.ReduceOp.AVG, group=group)          # (sync op: enqueued on `comm`, the host does not wait)
                else:
                    if dp["average"]:
                        s.mul_(1.0 / ws)
                    dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
                ops.cast_bf16_f32(s, t)
            ev = torch.cuda.Event()
            ev.record(comm)
        return [_Bf16WireWork(ev)]

    def _exchange(self, tensors, exposed=False):
        """``exposed``: nothing is left to overlap with (the final slices of a step) - the NVLS kernel then gets ``tail_ctas`` CTAs
        instead of the few that share the SMs with the backward."""
        dp = self._dp
        if not tensors:
            return []
        if dp.get("exchange") == "nvls":
            if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(dp["group"]) == 1:
                return []
            return self._nvls_exchange(tensors, dp["tail_ctas"] if exposed else None)
        if dp.get("wire") == "bf16":
            return self._bf16_wire_exchange(tensors)
        return allreduce_flat(tensors, dp["group"], dp["average"], async_op=True)

    @staticmethod
    def nvls_available(group=None, device=None):
        """Collective probe: True on every rank iff every rank can map a symmetric-memory buffer at a multicast (NVLS) address -
        what ``exchange="nvls"`` needs. Any failure on any rank -> False everywhere (callers fall back to NCCL)."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return False
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        try:
            import torch.distributed._symmetric_memory as symm
            t = symm.empty(4096, dtype=torch.float32, device=device)
            hdl = symm.rendezvous(t, group if group is not None else dist.group.WORLD)
            ok = 1 if hdl.multicast_ptr else 0
        except Exception:
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        return bool(int(flag.item()))

    def enable_overlapped_allreduce(self, group=None, average=True, cnn_buckets=False, exchange="nccl", max_ctas=None, wire="fp32", tail_ctas=132):
        """Start the all-reduce of the transformer gradient buffer (75 % of the payload) as soon as the last
        outstanding transformer backward of the step has finished, so that it overlaps the remaining CNN backward
        (what Horovod's background fusion thread did for the reference). ``allreduce_grads()`` then only exchanges
        the CNN buffer and joins. Safe inside CUDA-graph capture (ProcessGroupNCCL forks/joins its stream).

        ``cnn_buckets``: also exchange the tail of the CNN buffer (res5 + grid_encoder, 78 % of it) as soon as the
        res5 backward has enqueued its last weight gradient, leaving only res3/res4 (33 MB) for the final exchange.
        The collective is issued from the wgrad side stream, which is the stream those gradients are written on.
        ``wire="bf16"``: exchange the gradients as bf16 (see ``_bf16_wire_exchange``).
        ``max_ctas``: CTAs of the NVLS kernel while it overlaps the backward; ``None`` picks by world size - a rank reduces 1/world of
        the buffer, so two ranks need twice the CTAs of four to finish inside the CNN backward."""
        assert exchange in ("nccl", "nvls") and wire in ("fp32", "bf16")
        if not max_ctas:
            world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
            max_ctas = 64 if world <= 4 else 32
        self._dp = dict(group=group, average=average, works=[], tf_started=False, cnn_lo=None, sync=True, exchange=exchange,
                        max_ctas=int(max_ctas), tail_ctas=int(tail_ctas if tail_ctas else max_ctas), handles={}, wire=wire, shadows={})
        if exchange == "nvls":
            # ``exchange="nvls"``: this library's own all-reduce through the NVSwitch (csrc/nvls.cu) instead of NCCL. The flat
            # gradient buffers must then live in symmetric memory, so call this BEFORE the first forward (buffers that already
            # exist are dropped and rebuilt).
            import torch.distributed._symmetric_memory as symm
            from .params import FlatGroup
            FlatGroup.grad_factory = staticmethod(lambda n, dev: symm.empty(n, dtype=torch.float32, device=dev).zero_())
            for m in (self.transformer, self.cnn):
                m._flat = None

        def hook(flat_grad):
            if not self._dp["sync"]:
                return
            self._dp["works"] += self._exchange([flat_grad])
            self._dp["tf_started"] = True
        self.transformer._grad_ready_hook = hook

        def cnn_hook(flat_grad, lo, side_stream):
            if not self._dp["sync"]:
                return
            if side_stream is not None:
                with torch.cuda.stream(side_stream):
                    self._dp["works"] += self._exchange([flat_grad[lo:]])
            else:
                self._dp["works"] += self._exchange([flat_grad[lo:]])
            self._dp["cnn_lo"] = lo
        self.cnn._bucket_hook = cnn_hook if cnn_buckets else None

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient accumulation: inside this context backward passes only accumulate into the flat buffers - no hook starts
        an exchange and ``allreduce_grads()`` does nothing - so that the buffers are exchanged ONCE, by the last micro-step
        run outside it. (The reference synchronizes on every micro-step, src/tasks/run_video_retrieval.py:425-432: with
        ``gradient_accumulation_steps = k`` that is k times the traffic for the same result, SURVEY.md §8e.)"""
        dp = getattr(self, "_dp", None)
        if dp is None:
            dp = self._dp_nosync = dict(sync=True)
        prev, dp["sync"] = dp["sync"], False
        try:
            yield
        finally:
            dp["sync"] = prev

    def allreduce_grads(self, group=None, average=True, async_op=False):
        """Average the flat fp32 gradient buffers over the data-parallel group (NCCL) - the replacement of
        ``optimizer.synchronize()`` (src/tasks/run_video_retrieval.py:432)."""
        dp = getattr(self, "_dp", None)
        if dp is None:
            if not getattr(self, "_dp_nosync", dict(sync=True))["sync"]:
                return []
            return allreduce_flat(self.flat_grads(), group, average, async_op)
        if not dp["sync"]:
            return []
        works, dp["works"] = dp["works"], []
        tf_started, dp["tf_started"] = dp["tf_started"], False
        lo, dp["cnn_lo"] = dp["cnn_lo"], None
        rest = []
        tf = self.transformer._flat
        if not tf_started and tf is not None and tf.grad is not None:      # hook did not fire (e.g. transformer frozen)
            rest.append(tf.grad)
        cf = self.cnn._flat
        if cf is not None and cf.grad is not None:
            g = cf.grad if lo is None else cf.grad[:lo]                    # the tail [lo:) is already in flight (cnn_buckets)
            if g.numel():
                rest.append(g)
        works += self._exchange(rest, exposed=True)
        for w in works:
            w.wait()
        return []
