"""cb_attention_probs (the attention probabilities behind ClipBertBaseModel's output_attentions) timed with CUDA events, and an eval
bert(...) forward at 448 px with output_hidden_states / output_attentions off and on.

Per shape: median over `--rounds` rounds of `--reps` back-to-back calls, and the kernel's fraction of its lower bound =
(bytes of P written + Q and K read once) / 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth, for a card allowed 700 W) over
the measured time. The card name, power limit and max SM clock are read in the same run.
Usage: python tools/profile_attention_probs.py [--reps 50 --rounds 7 --out tool_out/attention_probs.txt]"""
import argparse
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

HEADS = 12
HBM_BYTES_PER_S = 3.35e12
# (sequences, L, Lt, what)
SHAPES = [(128, 41, 32, "224 px, 32-token captions"),
          (256, 69, 20, "MSRVTT retrieval 448 px"),
          (128, 149, 100, "DiDeMo / ActivityNet 448 px"),
          (80, 169, 25, "TGIF-QA 768 px"),
          (1, 521, 512, "512-token text, 224 px")]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return "%s | nvidia-smi name, power.limit, clocks.max.sm: %s" % (torch.cuda.get_device_name(0), q)


def timed(fn, reps, rounds):
    res = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) * 1e3 / reps)
    return statistics.median(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="tool_out/attention_probs.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    dev = torch.device("cuda:0")
    lines = ["card: " + card(),
             "cb_attention_probs, %d heads x 64, dropout 0.1; median of %d rounds of %d calls" % (HEADS, args.rounds, args.reps),
             "%-5s %-4s %-4s %10s %10s %12s %9s  %s" % ("nseq", "L", "Lt", "P MB", "time us", "bound us", "of bound", "configuration")]
    print("\n".join(lines), flush=True)
    for nseq, L, lt, what in SHAPES:
        g = torch.Generator().manual_seed(1)
        qkv = torch.randn(nseq * L, 3 * 768, generator=g).to(dev, torch.bfloat16)
        mask = torch.ones(nseq, lt, dtype=torch.int64, device=dev)
        mask[:, lt - lt // 4:] = 0
        ctx = torch.empty(nseq * L, 768, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(nseq, HEADS, L, device=dev)
        probs = torch.empty(nseq, HEADS, L, L, device=dev)
        ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 7)

        def run():
            ops.attention_probs(qkv, mask, lse, probs, nseq, L, lt, HEADS, 0.1, 7)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        us = timed(run, args.reps, args.rounds)
        p_bytes = 4 * nseq * HEADS * L * L
        bound = (p_bytes + 2 * 2 * nseq * L * 768) / HBM_BYTES_PER_S * 1e6
        line = "%-5d %-4d %-4d %10.1f %10.1f %12.1f %9.3f  %s" % (nseq, L, lt, p_bytes / 1e6, us, bound, bound / us, what)
        print(line, flush=True)
        lines.append(line)
        del qkv, ctx, lse, probs
        torch.cuda.empty_cache()
    # ---- eval bert(...) at 448 px (7 x 7 grid, 20-token captions: L = 69), flags off / on ----
    from oracle.clipbert_ref import BERT_CFG
    nseq, lt = 256, 20
    g = torch.Generator().manual_seed(2)
    grid = torch.randn(nseq, 1, 7, 7, 768, generator=g).to(dev, torch.bfloat16)
    ids = torch.randint(1000, 30000, (nseq, lt), generator=g).to(dev)
    mask = torch.ones(nseq, lt, dtype=torch.int64, device=dev)
    lines.append("eval bert(...) forward, %d sequences, L = %d (448 px), median of %d rounds of %d calls:" % (nseq, lt + 49, args.rounds, 10))
    for flags in (False, True):
        torch.manual_seed(0)
        cfg = types.SimpleNamespace(**dict(BERT_CFG, output_hidden_states=flags, output_attentions=flags))
        model = cb.ClipBertBaseModel(cfg).to(dev).eval()

        def fwd():
            with torch.no_grad():
                return model(ids, grid, mask)
        for _ in range(3):
            fwd()
        torch.cuda.synchronize()
        us = timed(fwd, 10, args.rounds)
        line = "  output_hidden_states = output_attentions = %-5s %10.1f us" % (flags, us)
        print(line, flush=True)
        lines.append(line)
        del model
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
