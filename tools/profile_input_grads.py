"""The gradient with respect to the input frames: cb_maxpool3x3s2_bwd_strided (the stem pool's backward + ReLU', on the
space-to-depth stem's grid) and cb_stem_dgrad (the 7x7/s2 transposed convolution to the frames) timed with CUDA events at the
headline shape (128 frames of 224 px) and at 448 px (32 frames), and an eval forward + backward to the frames through a fully
frozen ClipBert on the retrieval head at the headline shape (32 videos x 2 clips x 2 frames, forward_clips), against the same
forward with frames that do not require grad, with torch.cuda.max_memory_allocated for both.

The input stage: cb_resize_pad_bwd next to cb_resize_pad at decoded sizes users feed (720p, 240p, 1080p and 2160p sources),
and the same attribution pass from fp32 frames decoded at 1280 x 720, through input_stage.resize_pad to 224 px.

Per kernel: median over `--rounds` rounds of `--reps` back-to-back launches; compulsory bytes (pool: dy and x read, dx written
once; stem: dc1 read, fp32 frames written once; resize_pad: the source read, the padded frame written; resize_pad_bwd: the
new_h x new_w part of dy read, the source-sized dx written) over the time, and that as a fraction of 3.35 TB/s (the H100 SXM
data-sheet HBM3 bandwidth, for a card allowed 700 W). The card name, power limit and max SM clock are read in the same run.
Usage: python tools/profile_input_grads.py [--reps 20 --rounds 5 --out tool_out/input_grads.txt]"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = [(128, 224, "headline: 128 frames of 224 px"), (32, 448, "native resolution: 32 frames of 448 px")]
RESIZE_SHAPES = [(64, 720, 1280, 448), (64, 240, 320, 448), (16, 1080, 1920, 768), (16, 2160, 3840, 448)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "nvidia-smi unavailable"
    return "%s | nvidia-smi name, power.limit, clocks.max.sm: %s" % (torch.cuda.get_device_name(0), q)


def timed(fn, reps, rounds):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / reps)
    return statistics.median(ts)


def kernels(out, reps, rounds):
    from clipbert_b200 import ops
    import test_gpu_input_grads as IG
    dev = torch.device("cuda:0")
    w = IG.stem_operand(dev)
    for n, size, what in SHAPES:
        ho = (size - 1) // 2 + 1
        hh = (ho - 1) // 2 + 1
        hs = ho + 3
        x = torch.rand(n * hs * hs, 64, device=dev).to(torch.bfloat16)
        dy = torch.randn(n * hh * hh, 64, device=dev).to(torch.bfloat16)
        dc1 = torch.empty(n * ho * ho, 64, device=dev, dtype=torch.bfloat16)
        dx = torch.empty(n, 3, size, size, device=dev)
        t_pool = timed(lambda: ops.maxpool3x3s2_bwd(dy, x, dc1, n, ho, ho, 64, row_pitch=hs, img_pitch=hs * hs), reps, rounds)
        t_stem = timed(lambda: ops.stem_dgrad(dc1, w, dx, n, size, size), reps, rounds)
        b_pool = 2 * 64 * (n * hh * hh + 2 * n * ho * ho)
        b_stem = 2 * 64 * n * ho * ho + 4 * 3 * n * size * size
        flop = 2 * 3 * 64 * 49 * n * ho * ho
        for name, t, b in (("cb_maxpool3x3s2_bwd_strided", t_pool, b_pool), ("cb_stem_dgrad", t_stem, b_stem)):
            extra = " | %.1f TFLOP/s (%.2f GFLOP)" % (flop / t / 1e9, flop / 1e9) if name == "cb_stem_dgrad" else ""
            out("%-28s %-42s %8.3f ms  %7.1f MB  %6.2f TB/s  %5.1f %% of HBM bound%s" % (
                name, what, t, b / 1e6, b / t / 1e9, 100.0 * b / HBM_BYTES_PER_S / (t / 1e3), extra))


def resize_kernels(out, reps, rounds):
    from clipbert_b200 import input_stage, ops
    dev = torch.device("cuda:0")
    for n, h, w, size in RESIZE_SHAPES:
        nh, nw = input_stage.get_resize_size(h, w, size)
        x = torch.rand(n, 3, h, w, device=dev) * 255
        y = torch.empty(n, 3, size, size, device=dev)
        dy = torch.randn(n, 3, size, size, device=dev)
        dx = torch.empty_like(x)
        t_fwd = timed(lambda: ops.resize_pad(x, y, nh, nw), reps, rounds)
        t_bwd = timed(lambda: ops.resize_pad_bwd(dy, dx, nh, nw), reps, rounds)
        what = "%d frames %d x %d -> %d (%d x %d)" % (n, w, h, size, nw, nh)
        src, dst = 4 * n * 3 * h * w, 4 * n * 3 * size * size
        for name, t, b in (("cb_resize_pad", t_fwd, src + dst), ("cb_resize_pad_bwd", t_bwd, 4 * n * 3 * nh * nw + src)):
            out("%-28s %-42s %8.3f ms  %7.1f MB  %6.2f TB/s  %5.1f %% of HBM bound" % (
                name, what, t, b / 1e6, b / t / 1e9, 100.0 * b / HBM_BYTES_PER_S / (t / 1e3)))


def decoded_attribution(out, reps, rounds):
    """Eval forward + backward to fp32 frames decoded at 1280 x 720, through resize_pad to 224 px, on the fully frozen model."""
    import clipbert_b200 as cb
    from clipbert_b200 import input_stage
    from clipbert_b200.workload import IMAGE_MEAN
    from oracle import synth
    from util import make_cfg
    dev = torch.device("cuda:0")
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="R-50-grid.yaml")
    model.load_state_dict(synth.full_state_dict(42))
    model = model.to(dev).eval()
    for p in model.parameters():
        p.requires_grad_(False)
    input_stage.set_image_norm(model, IMAGE_MEAN)
    batch = synth.synth_batch(32, 4, n_ex=1, size=224, seed=1)
    mb = {k: (v.to(dev) if torch.is_tensor(v) else list(v)) for k, v in batch.items() if k != "visual_inputs"}
    decoded = torch.randint(0, 256, (32, 4, 3, 720, 1280), device=dev).float()

    def attribution():
        x = decoded.detach().requires_grad_(True)
        frames = input_stage.resize_pad(x, 224)
        score = model.forward_clips(dict(mb, visual_inputs=frames), 2)["logits"][..., 1].sum()
        return torch.autograd.grad(score, x)[0]

    attribution()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = timed(attribution, reps, rounds)
    out("%-40s 32 videos x 2 clips x 2 frames decoded at 1280 x 720 -> 224 px: %8.2f ms   max_memory_allocated %.2f GB" % (
        "eval forward + backward to decoded frames", t, torch.cuda.max_memory_allocated() / 1e9))


def end_to_end(out, reps, rounds):
    import clipbert_b200 as cb
    from oracle import synth
    from util import make_cfg
    dev = torch.device("cuda:0")
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="R-50-grid.yaml")
    model.load_state_dict(synth.full_state_dict(42))
    model = model.to(dev).eval()
    for p in model.parameters():
        p.requires_grad_(False)
    batch = synth.synth_batch(32, 4, n_ex=1, size=224, seed=1)
    mb = {k: (v.to(dev) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
    frames = mb["visual_inputs"]

    def plain():
        return model.forward_clips(dict(mb, visual_inputs=frames), 2)["logits"]

    def attribution():
        x = frames.detach().requires_grad_(True)
        score = model.forward_clips(dict(mb, visual_inputs=x), 2)["logits"][..., 1].sum()
        return torch.autograd.grad(score, x)[0]

    for name, fn in (("eval forward, frames without grad", plain), ("eval forward + backward to the frames", attribution)):
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t = timed(fn, reps, rounds)
        out("%-40s 32 videos x 2 clips x 2 frames, 224 px: %8.2f ms   max_memory_allocated %.2f GB" % (
            name, t, torch.cuda.max_memory_allocated() / 1e9))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_input_grads.py measures on the GPU"
    lines = []

    def out(s):
        print(s, flush=True)
        lines.append(s)
    out(card())
    kernels(out, args.reps, args.rounds)
    resize_kernels(out, args.reps, args.rounds)
    end_to_end(out, max(2, args.reps // 4), args.rounds)
    decoded_attribution(out, max(2, args.reps // 4), args.rounds)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
