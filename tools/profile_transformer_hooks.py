"""ClipBertBaseModel's module path (hooks on the transformer's modules) against the default path.

Eval bert(...) forward + backward (score on pooled_output, every parameter trainable, visual_inputs requiring grad) at 448 px
over 256 sequences (Lt 20, L = 69) and at 512 tokens over 8 sequences (L = 521), in four modes: no hooks (the default path);
observe-only forward hooks with a tensor hook on every encoder layer; the same on every hookable module below bert (every layer
split into its four sub-module nodes); and one 20-step integrated-gradients batch on bert.embeddings (forward-hook replacement and
torch.autograd.grad per step; its time is for all 20 steps). Median over `--rounds` rounds of `--reps` steps (CUDA events). Then
the word-vector text-embedding kernels against the id-based ones at the same shapes: cb_embed_text_fwd_vectors against
cb_embed_text_fwd, and cb_embed_text_bwd_vectors (+ cb_embed_word_scatter) against cb_embed_text_bwd, default mode, with the
fraction of the HBM lower bound (compulsory bytes / 3.35 TB/s, the H100 SXM data-sheet bandwidth for a 700 W card). The card
name, power limit and max SM clock are read in the same run.
Usage: python tools/profile_transformer_hooks.py [--reps 10 --rounds 5 --out tool_out/transformer_hooks.txt]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from profile_attention_probs import HBM_BYTES_PER_S, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="tool_out/transformer_hooks.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    import clipbert_b200 as cb
    from clipbert_b200.modeling import _BERT_SITES
    from oracle import synth
    from util import make_cfg
    dev = torch.device("cuda:0")
    lines = ["card: " + card()]

    def emit(s):
        print(s, flush=True)
        lines.append(s)
    sd = synth.full_state_dict(42)
    bert = cb.ClipBertBaseModel(make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0))
    bert.load_state_dict({k[len("transformer.bert."):]: v for k, v in sd.items() if k.startswith("transformer.bert.")})
    bert = bert.to(dev).eval()
    layers = list(bert.encoder.layer)
    every = [m for m in bert.modules() if isinstance(m, _BERT_SITES) and m is not bert]
    for name, nseq, lt, gh in (("448 px", 256, 20, 7), ("512 tokens", 8, 512, 3)):
        g = torch.Generator().manual_seed(1)
        grid = torch.randn(nseq, 2, gh, gh, 768, generator=g).abs().to(dev, torch.bfloat16)
        ids, mask = synth.synth_text(nseq, lt, seed=2)
        ids, mask = ids.to(dev), mask.to(dev)
        w = torch.randn(nseq, 768, generator=g).to(dev)
        emit("eval bert(...) forward + backward, %s: %d sequences, L = %d, median of %d rounds of %d steps:"
             % (name, nseq, lt + gh * gh, args.rounds, args.reps))

        def step():
            gc = grid.clone().requires_grad_(True)
            (bert(ids, gc, mask)[1].float() * w).sum().backward()
        for mode, mods in (("no hooks", []), ("hooks on every layer", layers), ("hooks on every sub-module", every)):
            kept = {}

            def fh(mod, i, o, kept=kept):
                t = o[0] if isinstance(o, tuple) else o
                kept[id(mod)] = t
                t.register_hook(lambda g_: kept.__setitem__(-id(mod), g_))
            handles = [m.register_forward_hook(fh) for m in mods]
            for _ in range(2):
                step()
            torch.cuda.synchronize()
            emit("  %-30s %10.1f us" % (mode, timed(step, args.reps, args.rounds)))
            for h in handles:
                h.remove()
        saved = {}
        h = bert.embeddings.register_forward_hook(lambda m, i, o: saved.__setitem__("x", o.detach().float()))
        with torch.no_grad():
            bert(ids, grid, mask)
        h.remove()

        def ig():
            x, total = saved["x"], None
            for k in range(1, 21):
                xk = (x * (k / 20)).requires_grad_(True)
                hk = bert.embeddings.register_forward_hook(lambda m, i, o: xk)
                (gk,) = torch.autograd.grad((bert(ids, grid, mask)[1].float() * w).sum(), xk)
                hk.remove()
                total = gk if total is None else total + gk
            return x * total / 20
        ig()
        torch.cuda.synchronize()
        emit("  %-30s %10.1f us" % ("integrated gradients, 20 steps", timed(ig, 1, args.rounds)))
    from clipbert_b200 import ops
    emit("text embeddings, ids against word vectors, median of %d rounds of %d calls:" % (args.rounds, args.reps * 5))
    emit("%-22s %-30s %10s %10s %9s" % ("nseq x lt", "kernel", "time us", "bound us", "of bound"))
    H = 768
    for nseq, lt in ((256, 20), (8, 512)):
        g = torch.Generator().manual_seed(lt)
        R, L = nseq * lt, lt + 49
        word = torch.randn(30522, H, generator=g).to(dev)
        ids = torch.randint(0, 30522, (nseq, lt), generator=g).to(dev)
        vec = word[ids.reshape(-1)].contiguous()
        pos, typ = torch.randn(lt, H, generator=g).to(dev), torch.randn(1, H, generator=g).to(dev)
        gam, bet = torch.ones(H, device=dev), torch.zeros(H, device=dev)
        out, stats = torch.empty(nseq * L, H, dtype=torch.bfloat16, device=dev), torch.empty(R, 2, device=dev)
        dh = torch.randn(nseq * L, H, generator=g).to(dev, torch.bfloat16)
        dvec, dword = torch.empty(R, H, device=dev), torch.zeros_like(word)
        tabs = [torch.zeros_like(t) for t in (pos, typ, gam, bet)]
        fwd_bytes = R * H * (4 + 2) + R * 8                       # vectors / rows read, bf16 rows written, stats
        bwd_bytes = R * H * (2 + 4 + 4) + R * 8                   # d rows read, vectors read, d vectors written, stats
        for name, fn, nbytes in (
                ("cb_embed_text_fwd", lambda: ops.embed_text_fwd(ids, word, pos, typ, gam, bet, out, stats, nseq, lt, L, 1e-12, 0.1, 1),
                 fwd_bytes),
                ("cb_embed_text_fwd_vectors", lambda: ops.embed_text_fwd_vectors(vec, pos, typ, gam, bet, out, stats, nseq, lt, L, 1e-12,
                                                                                 0.1, 1), fwd_bytes),
                ("cb_embed_text_bwd", lambda: ops.embed_text_bwd(dh, ids, word, pos, typ, gam, stats, dword, *tabs, nseq, lt, L, 0.1, 1),
                 bwd_bytes),
                ("cb_embed_text_bwd_vectors", lambda: ops.embed_text_bwd_vectors(dh, vec, pos, typ, gam, stats, dvec, *tabs, nseq, lt,
                                                                                 L, 0.1, 1), bwd_bytes),
                ("  + cb_embed_word_scatter", lambda: ops.embed_word_scatter(ids, dvec, dword), R * H * 12)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            us = timed(fn, args.reps * 5, args.rounds)
            bound = nbytes / HBM_BYTES_PER_S * 1e6
            emit("%-22s %-30s %10.1f %10.1f %9.3f" % ("%d x %d" % (nseq, lt), name, us, bound, bound / us))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
