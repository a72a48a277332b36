"""Checkpoint key layouts of the reference, into and out of the H100 modules (SURVEY.md §8 f4).

Mirrors the three entry points the reference task scripts use to get weights into ``ClipBert``
(src/tasks/run_video_retrieval.py:202-210):

  load_state_dict_with_mismatch(model, state_dict_or_path)   src/utils/load_save.py:71-100 - e2e / BERT checkpoints: keys that are
        missing on either side or whose shape differs (task heads with another num_labels) are skipped, never an error
  convert_torchvision_ckpt_to_detectron2(ckpt_or_path)       src/utils/load_save.py:318-363 - torchvision ResNet names -> d2 names
  load_detectron2_checkpoint(backbone, path_or_dict)         what ``GridFeatBackbone.load_state_dict(path)`` (grid_feat.py:72-80) gets
        from d2's DetectionCheckpointer for ``grid_feat_R-50.pth``: a ``{"model": {...}}`` (or flat) dict keyed relative to
        ``cnn.feature`` (``backbone.stem.conv1.weight`` ...), torch tensors or numpy arrays; the dead RPN / ROI-head keys are ignored

and ``export_state_dict(model)`` for the way back: contiguous CPU tensors under the reference's keys (the live parameters are
views into flat fp32 buffers, conv weights physically KRSC). Host logic only - no kernels; loading marks the bf16 tensor-core
operands stale so the next forward re-casts them.
"""
import pickle
from typing import Any, Dict

import torch

TORCHVISION_TO_D2 = {            # load_save.py:335-345, applied in this order as substring replacements
    "layer1": "res2",
    "layer2": "res3",
    "layer3": "res4",
    "layer4": "res5",
    "bn1": "conv1.norm",
    "bn2": "conv2.norm",
    "bn3": "conv3.norm",
    "downsample.0": "shortcut",
    "downsample.1": "shortcut.norm",
}


def _load_file(path):
    if str(path).endswith(".pkl"):
        with open(path, "rb") as f:
            return pickle.load(f, encoding="latin1")
    return torch.load(path, map_location="cpu")


def _mark_updated(model):
    for m in model.modules():
        if hasattr(m, "mark_weights_updated"):
            m.mark_weights_updated()


def load_state_dict_with_mismatch(model, loaded_state_dict_or_path):
    """In place, like the reference. Returns dict(loaded=[...], unexpected=[...], missing=[...], mismatched=[...]) (the reference
    only logs these four sets)."""
    loaded = _load_file(loaded_state_dict_or_path) if isinstance(loaded_state_dict_or_path, str) else loaded_state_dict_or_path
    own = model.state_dict()
    model_keys, load_keys = set(own.keys()), set(loaded.keys())
    toload, mismatched = {}, []
    for k in model_keys:
        if k in load_keys:
            if own[k].shape != loaded[k].shape:
                mismatched.append(k)
            else:
                toload[k] = loaded[k]
    model.load_state_dict(toload, strict=False)
    _mark_updated(model)
    return dict(loaded=sorted(toload), unexpected=sorted(load_keys - model_keys), missing=sorted(model_keys - load_keys),
                mismatched=sorted(mismatched))


def convert_torchvision_ckpt_to_detectron2(ckpt_or_path) -> Dict[str, Any]:
    """torchvision ResNet state dict (or its path) -> ``{"model": d2-named dict, "__author__", "matching_heuristics"}``."""
    sd = _load_file(ckpt_or_path) if isinstance(ckpt_or_path, str) else ckpt_or_path
    out = {}
    for name, param in sd.items():
        for old, new in TORCHVISION_TO_D2.items():
            name = name.replace(old, new)
        if not name.startswith("res"):          # first conv / bn (and fc) live under "stem."
            name = "stem." + name
        out[name] = param
    return {"model": out, "__author__": "clipbert_b200", "matching_heuristics": True}


def load_detectron2_checkpoint(backbone, path_or_dict):
    """``backbone``: a GridFeatBackbone. Accepts d2 checkpoints keyed ``backbone.res4.0.conv1.weight`` (relative to ``feature``),
    bare ResNet keys (``res4.0.conv1.weight`` / ``stem.conv1.weight``, the output of convert_torchvision_ckpt_to_detectron2), or
    full ``cnn.``-/``feature.``-prefixed keys. Returns (loaded, ignored) key lists; shapes must match (a backbone has no task heads)."""
    ck = _load_file(path_or_dict) if isinstance(path_or_dict, str) else path_or_dict
    ck = ck.get("model", ck)
    own = backbone.state_dict()
    loaded, ignored, toload = [], [], {}
    for k, v in ck.items():
        v = v if torch.is_tensor(v) else torch.as_tensor(v)
        cands = (k, "feature." + k, "feature.backbone." + k, k[len("cnn."):] if k.startswith("cnn.") else None)
        hit = next((c for c in cands if c is not None and c in own), None)
        if hit is None:
            ignored.append(k)            # fc.*, num_batches_tracked, proposal_generator.*, roi_heads.*, pixel_mean ...
            continue
        if tuple(own[hit].shape) != tuple(v.shape):
            raise ValueError("shape mismatch for %s: checkpoint %s, model %s" % (k, tuple(v.shape), tuple(own[hit].shape)))
        toload[hit] = v
        loaded.append(hit)
    torch.nn.Module.load_state_dict(backbone, toload, strict=False)
    backbone.mark_weights_updated()
    return sorted(loaded), sorted(ignored)


def export_state_dict(model):
    """Reference-keyed, contiguous, CPU copy of the model's parameters and buffers (what ModelSaver / the restorer write)."""
    return {k: v.detach().to("cpu").contiguous().clone() for k, v in model.state_dict().items()}
