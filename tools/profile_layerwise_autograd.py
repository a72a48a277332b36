"""cb_attention_bwd_dv (the value gradient of the attention backward alone, for ClipBertBaseModel.layerwise_autograd's split at a
differentiable map) timed with CUDA events at the five shapes of tools/profile_attention_probs.py, and an eval bert(...) forward +
backward at 448 px on 256 sequences in three modes: the default (one autograd node), layerwise_autograd on, and layerwise_autograd
on with a tensor hook on all 12 attention maps.

Per shape: median over `--rounds` rounds of `--reps` back-to-back calls, and the kernel's fraction of its HBM lower bound =
compulsory bytes / 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth, for a card allowed 700 W) over the measured time.
Compulsory bytes: Q, K and dO read once, dV written, lse read (the kernel rebuilds P and never reads a map). The card name, power
limit and max SM clock are read in the same run.
Usage: python tools/profile_layerwise_autograd.py [--reps 50 --rounds 7 --out tool_out/layerwise_autograd.txt]"""
import argparse
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from profile_attention_probs import HBM_BYTES_PER_S, HEADS, SHAPES, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="tool_out/layerwise_autograd.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    dev = torch.device("cuda:0")
    lines = ["card: " + card(),
             "cb_attention_bwd_dv, %d heads x 64, dropout 0.1; median of %d rounds of %d calls" % (HEADS, args.rounds, args.reps),
             "%-5s %-4s %-4s %10s %10s %9s %12s  %s" % ("nseq", "L", "Lt", "time us", "bound us", "of bound", "attn_bwd us", "configuration")]
    print("\n".join(lines), flush=True)
    for nseq, L, lt, what in SHAPES:
        g = torch.Generator().manual_seed(1)
        qkv = torch.randn(nseq * L, 3 * 768, generator=g).to(dev, torch.bfloat16)
        dctx = torch.randn(nseq * L, 768, generator=g).to(dev, torch.bfloat16)
        mask = torch.ones(nseq, lt, dtype=torch.int64, device=dev)
        mask[:, lt - lt // 4:] = 0
        ctx = torch.empty(nseq * L, 768, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(nseq, HEADS, L, device=dev)
        dqkv = torch.zeros(nseq * L, 3 * 768, device=dev, dtype=torch.bfloat16)
        ops.attention_fwd(qkv, mask, ctx, lse, nseq, L, lt, HEADS, 0.1, 7)

        def run_dv():
            ops.attention_bwd_dv(qkv, mask, lse, dctx, dqkv, nseq, L, lt, HEADS, 0.1, 7)

        def run_ab():
            ops.attention_bwd(qkv, mask, ctx, dctx, lse, dqkv, nseq, L, lt, HEADS, 0.1, 7)
        for _ in range(3):
            run_dv()
            run_ab()
        torch.cuda.synchronize()
        us = timed(run_dv, args.reps, args.rounds)
        us_ab = timed(run_ab, args.reps, args.rounds)
        nbytes = 2 * nseq * L * 768 * 4 + 4 * nseq * HEADS * L      # Q, K, dO read, dV written (bf16), lse read
        bound = nbytes / HBM_BYTES_PER_S * 1e6
        line = "%-5d %-4d %-4d %10.1f %10.1f %9.3f %12.1f  %s" % (nseq, L, lt, us, bound, bound / us, us_ab, what)
        print(line, flush=True)
        lines.append(line)
        del qkv, dctx, ctx, lse, dqkv
        torch.cuda.empty_cache()
    # ---- eval bert(...) forward + backward at 448 px (7 x 7 grid, 20-token captions: L = 69) ----
    from oracle.clipbert_ref import BERT_CFG
    nseq, lt = 256, 20
    L = lt + 49
    g = torch.Generator().manual_seed(2)
    grid = torch.randn(nseq, 1, 7, 7, 768, generator=g).to(dev, torch.bfloat16)
    ids = torch.randint(1000, 30000, (nseq, lt), generator=g).to(dev)
    mask = torch.ones(nseq, lt, dtype=torch.int64, device=dev)
    w_pool = torch.randn(nseq, 768, generator=g).to(dev)
    head = ("eval bert(...) forward + backward, %d sequences, L = %d (448 px), both output flags and differentiable_attentions on, "
            "score on pooled_output, median of %d rounds of %d steps:" % (nseq, L, args.rounds, 5))
    print(head, flush=True)
    lines.append(head)
    torch.manual_seed(0)
    cfg = types.SimpleNamespace(**dict(BERT_CFG, output_hidden_states=True, output_attentions=True))
    model = cb.ClipBertBaseModel(cfg).to(dev).eval()
    model.differentiable_attentions = True
    saved = {}
    for mode in ("default", "layerwise_autograd", "layerwise_autograd + hooks on 12 maps"):
        model.layerwise_autograd = mode != "default"

        def step():
            seq, pooled, hidden, attn = model(ids, grid, mask)
            if "hooks" in mode:
                for i, a in enumerate(attn):
                    a.register_hook(lambda gr, i=i: saved.__setitem__(i, gr))
            (pooled.float() * w_pool).sum().backward()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        us = timed(step, 5, args.rounds)
        line = "  %-40s %10.1f us" % (mode, us)
        print(line, flush=True)
        lines.append(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
