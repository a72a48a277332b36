"""Attention backward for sequences longer than 64 tokens: the tensor-core kernels (attn_tc_bwd_kv_kernel / attn_tc_bwd_q_kernel)
against the CUDA-core kernels (cb_debug_attention_general(1)), alternating in one session, at the shapes of the reference's
native-resolution training configurations. CUDA events around `--reps` back-to-back calls, `--rounds` rounds per path; the
median round is reported. Also prints the card name, power limit and SM clock, and the relative difference of the two paths'
dQKV. Writes tool_out/attention_bwd.txt. Usage: python tools/profile_attention.py [--reps 50 --rounds 7]"""
import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

HEADS = 12
# (sequences per step, L, Lt, what): the reference's configurations at 448 / 768 px (src/configs/*.json)
SHAPES = [(256, 69, 20, "MSRVTT retrieval 448 px: 16 videos x 8 clips x (pos + neg)"),
          (128, 149, 100, "DiDeMo / ActivityNet retrieval, MSRVTT-QA 448 px"),
          (80, 169, 25, "TGIF-QA 768 px"),
          (64, 164, 20, "VQA 768 px"),
          (1, 521, 512, "512-token text, 224 px")]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return "%s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="tool_out/attention_bwd.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    from clipbert_b200 import _lib, ops
    lib = _lib.lib()
    dev = torch.device("cuda:0")
    lines = ["card: " + card(), "cb_attention_bwd, 12 heads x 64, dropout 0.1; %d calls per round, median of %d rounds per path, "
             "paths alternating" % (args.reps, args.rounds),
             "%-5s %-4s %-4s %12s %12s %8s %10s  %s" % ("nseq", "L", "Lt", "CUDA-core us", "tensor us", "speed-up", "relerr", "configuration")]
    print("\n".join(lines), flush=True)
    for nseq, L, lt, what in SHAPES:
        g = torch.Generator().manual_seed(1)
        qkv = torch.randn(nseq * L, 3 * 768, generator=g).to(dev, torch.bfloat16)
        dctx = torch.randn(nseq * L, 768, generator=g).to(dev, torch.bfloat16)
        mask = torch.ones(nseq, lt, dtype=torch.int64, device=dev)
        mask[:, lt - lt // 4:] = 0
        ctx = torch.empty(nseq * L, 768, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(nseq, HEADS, L, device=dev)
        ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 7)
        out = {1: torch.empty_like(qkv), 0: torch.empty_like(qkv)}
        times = {1: [], 0: []}
        try:
            for general in (1, 0):      # warm-up: module load, first launches
                lib.cb_debug_attention_general(ctypes.c_int(general))
                for _ in range(5):
                    ops.attention_bwd(qkv, mask, ctx, dctx, lse, out[general], nseq, L, lt, HEADS, 0.1, 7)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for general in (1, 0):
                    lib.cb_debug_attention_general(ctypes.c_int(general))
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        ops.attention_bwd(qkv, mask, ctx, dctx, lse, out[general], nseq, L, lt, HEADS, 0.1, 7)
                    e1.record()
                    e1.synchronize()
                    times[general].append(1e3 * e0.elapsed_time(e1) / args.reps)
        finally:
            lib.cb_debug_attention_general(ctypes.c_int(0))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        a, b = out[0].double(), out[1].double()
        err = float((a - b).norm() / b.norm())
        line = "%-5d %-4d %-4d %12.1f %12.1f %7.2fx %10.2e  %s (spread %.1f-%.1f / %.1f-%.1f us)" % (
            nseq, L, lt, med[1], med[0], med[1] / med[0], err, what, min(times[1]), max(times[1]), min(times[0]), max(times[0]))
        lines.append(line)
        print(line, flush=True)
        del qkv, dctx, ctx, lse, out
    lines.append("card after: " + card())
    print(lines[-1])
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    open(args.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
