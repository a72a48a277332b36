"""GridFeatBackbone's module path (hooks on the CNN's modules) against the default path, and cb_nhwc_intake alone.

Eval pass: every CNN parameter frozen (grid_encoder included), frames that require grad, forward + backward to the
frames, 8 frames at 224 px and 4 at 448 px, in three modes: no hooks (the default path), a Grad-CAM forward + tensor hook on
res5[-1] (the module path), and the same hooks on all 16 blocks. Median over `--rounds` rounds of `--reps` steps (CUDA events).

cb_nhwc_intake: the masked intake of a block-output gradient (bf16 channels-last in, bf16 act, compact out) at the res2..res5
output shapes of the 224-px eval pass, and the fp32 contiguous-NCHW and generic-stride paths at the res4 shape. Its fraction of
the HBM lower bound = compulsory bytes (x read, act read, out written, once each) / 3.35 TB/s (the H100 SXM data-sheet HBM3
bandwidth, for a card allowed 700 W) over the measured time. The card name, power limit and max SM clock are read in the same run.
Usage: python tools/profile_cnn_hooks.py [--reps 20 --rounds 7 --out tool_out/cnn_hooks.txt]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from profile_attention_probs import HBM_BYTES_PER_S, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="tool_out/cnn_hooks.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from oracle import synth
    dev = torch.device("cuda:0")
    lines = ["card: " + card()]

    def emit(s):
        print(s, flush=True)
        lines.append(s)
    emit("cb_nhwc_intake, median of %d rounds of %d calls" % (args.rounds, args.reps * 5))
    emit("%-26s %-10s %10s %10s %9s" % ("shape (n, c, h, w)", "path", "time us", "bound us", "of bound"))
    for (n, c, h, w), path in (((8, 256, 56, 56), "cl+mask"), ((8, 512, 28, 28), "cl+mask"), ((8, 1024, 14, 14), "cl+mask"),
                               ((8, 2048, 7, 7), "cl+mask"), ((8, 1024, 14, 14), "nchw fp32"), ((8, 1024, 14, 14), "generic")):
        g = torch.Generator().manual_seed(c)
        if path == "cl+mask":
            x = torch.randn(n, c, h, w, generator=g).to(dev, torch.bfloat16).contiguous(memory_format=torch.channels_last)
            act = torch.randn(n * h * w, c, generator=g).to(dev, torch.bfloat16)
        elif path == "nchw fp32":
            x, act = torch.randn(n, c, h, w, generator=g).to(dev), None
        else:
            x, act = torch.randn(n, h, c, w, generator=g).to(dev, torch.bfloat16).permute(0, 2, 1, 3), None
        out = torch.empty(n * h * w, c, dtype=torch.bfloat16, device=dev)

        def run():
            ops.nhwc_intake(x, out, act=act)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        us = timed(run, args.reps * 5, args.rounds)
        nbytes = x.numel() * x.element_size() + out.numel() * 2 + (act.numel() * 2 if act is not None else 0)
        bound = nbytes / HBM_BYTES_PER_S * 1e6
        emit("%-26s %-10s %10.1f %10.1f %9.3f" % ((n, c, h, w), path, us, bound, bound / us))
    sd = synth.cnn_state_dict(42)
    for size, frames in ((224, 8), (448, 4)):
        m = cb.GridFeatBackbone()
        m.load_state_dict(sd)
        m = m.to(dev).eval()
        for p in m.parameters():
            p.requires_grad_(False)
        x = synth.synth_images(1, frames, size=size, seed=1).to(dev)
        emit("eval forward + backward to the frames, %d frames at %d px, all parameters frozen, median of %d rounds of %d steps:"
             % (frames, size, args.rounds, args.reps))
        blocks = [b for s in ("res2", "res3", "res4", "res5") for b in getattr(m.feature.backbone, s)]
        for mode, mods in (("no hooks", []), ("Grad-CAM hooks on res5[-1]", blocks[-1:]), ("hooks on all 16 blocks", blocks)):
            kept = {}

            def fh(mod, i, o):
                kept[id(mod)] = o
                o.register_hook(lambda g_: kept.__setitem__(-id(mod), g_))
            handles = [mod.register_forward_hook(fh) for mod in mods]

            def step():
                xg = x.clone().requires_grad_(True)
                m(xg).float().sum().backward()
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            us = timed(step, args.reps, args.rounds)
            emit("  %-30s %10.1f us" % (mode, us))
            for hd in handles:
                hd.remove()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
