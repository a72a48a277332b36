"""Helpers shared by the model-level GPU tests and tools/parity_report.py."""
import torch


def cnn_relu_masks(stash, prefix="cnn.feature.backbone."):
    """ReLU activation patterns of an H100 forward (from its backward stash) as oracle-side NCHW bool masks."""
    n = stash["n"]
    masks = {}
    for st in stash["blocks"]:
        h, w = st["h"], st["w"]
        p = prefix + st["name"] + "."
        a = st["a_pad"].view(n, h + 2, w + 2, -1)[:, 1:-1, 1:-1]
        b = st["b"].view(n, h, w, -1)
        y = st["y"]
        y = y.view(n, h + 2, w + 2, -1)[:, 1:-1, 1:-1] if y.shape[0] == n * (h + 2) * (w + 2) else y.view(n, h, w, -1)
        for site, t in (("conv1", a), ("conv2", b), ("out", y)):
            masks[p + site] = (t > 0).permute(0, 3, 1, 2).cpu()
    return masks


def cnn_patterns(stash, grid, prefix="cnn."):
    """Rounding object carrying the ReLU pattern and the max-pool selection of an H100 CNN forward."""
    import torch.nn.functional as F
    from oracle import clipbert_ref as R
    n, h, w = stash["n"], stash["h"], stash["w"]
    masks = cnn_relu_masks(stash, prefix + "feature.backbone.")
    c = grid.shape[-1]
    masks[prefix + "grid_encoder"] = (grid.detach() > 0).reshape(n, grid.shape[2], grid.shape[3], c).permute(0, 3, 1, 2).cpu()
    rnd = R.Rounding(relu_masks=masks)
    gconv = stash["gconv"].float().view(n, h, w, c).permute(0, 3, 1, 2).cpu()
    rnd.pool_indices = F.max_pool2d(gconv, 2, 2, return_indices=True)[1]
    return rnd
