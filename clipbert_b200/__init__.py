"""clipbert_b200 — the ClipBERT forward/backward hot path as hand-written sm_90a kernels.

Only what the path needs: ``csrc/`` (CUDA kernels + C ABI), ``_lib``/``ops`` (ctypes binding) and the
host-side mirrors of the reference module interface (``ClipBert``, ``GridFeatBackbone``,
``ClipBertFor*``). There is no CPU or eager-PyTorch fallback.
"""
from .e2e_model import ClipBert, clip_lse_loss, clip_pool_loss  # noqa: F401
from .grid_feat import GridFeatBackbone  # noqa: F401
from .modeling import (ClipBertBaseModel, ClipBertForMultipleChoice, ClipBertForPreTraining, ClipBertForRegression,  # noqa: F401
                       ClipBertForSequenceClassification, ClipBertForVideoTextRetrieval)
