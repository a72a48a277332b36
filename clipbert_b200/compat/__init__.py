"""Import-time stand-ins for the two third-party packages the reference task scripts import around the hot path and
that an H100 installation does not need (SURVEY.md §8b): ``horovod.torch`` (-> torch.distributed / NCCL) and ``apex``
(``amp`` is a no-op here: parameters stay fp32 masters and the kernels consume their own bf16 copy; ``FusedLayerNorm``
is only a parameter container on this path).

    import clipbert_b200.compat as compat
    compat.install()            # registers horovod / horovod.torch / apex / apex.amp / apex.normalization.* if absent
    import horovod.torch as hvd # now the module below

Only the calls the reference makes are provided (``grep -rn "hvd\\.\\|amp\\." src/``): nothing more.
"""
import sys
import types

from . import amp, horovod_torch


def alias_reference_modules():
    """Make the reference's own import lines resolve to this package (src/tasks/run_*.py:7-11, src/pretrain/run_pretrain.py:7-8):
    ``from src.modeling.e2e_model import ClipBert``, ``from src.modeling.modeling import ClipBertFor...`` and
    ``from src.modeling.grid_feat import GridFeatBackbone`` then import the H100 modules - the scripts stay byte-identical.
    Call it before the script's imports run, with the reference root on ``sys.path`` (its ``src`` package must be importable)."""
    import clipbert_b200.e2e_model as e2e
    import clipbert_b200.grid_feat as gf
    import clipbert_b200.modeling as mod
    sys.modules["src.modeling.e2e_model"] = e2e
    sys.modules["src.modeling.modeling"] = mod
    sys.modules["src.modeling.grid_feat"] = gf
    return ["src.modeling.e2e_model", "src.modeling.modeling", "src.modeling.grid_feat"]


def install(force=False):
    """Register the stand-ins under the names the reference imports. Real installations win unless ``force``."""
    def have(name):
        if name in sys.modules:
            return True
        import importlib.util
        try:
            return importlib.util.find_spec(name) is not None
        except (ImportError, ValueError):
            return False

    done = []
    if force or not have("horovod"):
        pkg = types.ModuleType("horovod")
        pkg.torch = horovod_torch
        sys.modules["horovod"] = pkg
        sys.modules["horovod.torch"] = horovod_torch
        done.append("horovod.torch")
    if force or not have("apex"):
        from torch import nn
        pkg = types.ModuleType("apex")
        norm = types.ModuleType("apex.normalization")
        fln = types.ModuleType("apex.normalization.fused_layer_norm")
        fln.FusedLayerNorm = nn.LayerNorm
        norm.fused_layer_norm = fln
        norm.FusedLayerNorm = nn.LayerNorm
        pkg.amp, pkg.normalization = amp, norm
        sys.modules.update({"apex": pkg, "apex.amp": amp, "apex.normalization": norm, "apex.normalization.fused_layer_norm": fln})
        done.append("apex")
    return done
