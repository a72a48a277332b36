"""``apex.amp`` as the reference uses it (src/tasks/run_video_retrieval.py:307-309,428-431,477-480; src/utils/load_save.py:
initialize / scale_loss / master_params / state_dict / load_state_dict). On the H100 path mixed precision is internal to the
kernels (fp32 master parameters, bf16 operand copies, fp32 accumulation, bf16 has fp32's exponent range: no loss scaling),
so every call is the identity."""
import contextlib


def initialize(models, optimizers=None, enabled=True, opt_level="O2", **_kw):
    return models if optimizers is None else (models, optimizers)


@contextlib.contextmanager
def scale_loss(loss, optimizers, delay_unscale=False, **_kw):
    yield loss


def master_params(optimizer):
    for group in optimizer.param_groups:
        for p in group["params"]:
            yield p


def state_dict(destination=None):
    return {} if destination is None else destination


def load_state_dict(state_dict):
    return None
