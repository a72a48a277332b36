"""Per-stage parity numbers of the H100 path against the CPU oracle (needs a GPU); written to a text report."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from model_util import cnn_patterns  # noqa: E402
from util import cosine, make_cfg, relerr  # noqa: E402


def main():
    import clipbert_b200 as cb
    from oracle import clipbert_ref as R, synth
    lines = []

    def out(*a):
        s = " ".join(str(x) for x in a)
        print(s, flush=True)
        lines.append(s)

    dev = torch.device("cuda:0")
    sd0 = synth.full_state_dict(42)
    cfg = make_cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = cb.ClipBert(cfg, detectron2_model_cfg="x").to(dev)
    model.load_state_dict(sd0)
    model.train()

    # ---------------- CNN forward ----------------
    x = synth.synth_images(2, 2, size=224, seed=5)
    with torch.no_grad():
        _, st32 = R.grid_feat_backbone(x, sd0, return_stages=True)
        _, st16 = R.grid_feat_backbone(x, sd0, return_stages=True, rnd=R.Rounding.bf16())
    model.cnn._capture = {}
    grid = model.cnn(x.to(dev))
    cap = model.cnn._capture
    out("== CNN forward (2x2 frames 224x224): relerr vs bf16-matched oracle | vs fp32 oracle")
    for name in ("stem", "res2", "res3", "res4", "res5"):
        got = cap[name].float().permute(0, 3, 1, 2)
        out("  %-6s %.3e | %.3e" % (name, relerr(got, st16[name]), relerr(got, st32[name])))
    out("  %-6s %.3e | %.3e" % ("grid", relerr(grid, st16["grid"]), relerr(grid, st32["grid"])))

    # ---------------- CNN backward with the run's own ReLU pattern ----------------
    pat = cnn_patterns(cap["stash"], grid)
    g = torch.Generator().manual_seed(1)
    dgrid = torch.randn(grid.shape, generator=g).to(torch.bfloat16).float()
    for label, rnd in (("fp32 oracle, own ReLU pattern", R.Rounding()), ("fp32 oracle, run's ReLU/max-pool pattern", pat)):
        sd = {k: (v.clone().requires_grad_(True) if (k.startswith("cnn.") and k.endswith(".weight") and "norm" not in k) else v)
              for k, v in sd0.items()}
        ref = R.grid_feat_backbone(x, sd, rnd=rnd)
        ref.backward(dgrid)
        if label.startswith("fp32 oracle, own"):
            model.cnn.zero_grad()
            model.zero_grad()
            grid.backward(dgrid.to(dev).to(grid.dtype), retain_graph=False)
        out("== CNN backward: gradient relerr / cosine vs " + label)
        for name, p in model.cnn.named_parameters():
            if not p.requires_grad:
                continue
            r = sd["cnn." + name].grad
            out("  %-48s %.3e  %.6f" % (name, relerr(p.grad, r), cosine(p.grad, r)))
    model.cnn._capture = None

    # ---------------- transformer ----------------
    tr = model.transformer
    nvid, T, n_ex = 3, 2, 2
    g = torch.Generator().manual_seed(2)
    gridt = (torch.randn(nvid, T, 3, 3, 768, generator=g).abs() * 2).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nvid * n_ex, 32, seed=3)
    labels = torch.randint(0, 2, (nvid * n_ex,), generator=g)
    sd = {k: (v.clone().requires_grad_(True) if k.startswith("transformer.") else v) for k, v in sd0.items()}
    gr = gridt.clone().requires_grad_(True)
    rep = R.repeat_tensor_rows(gr, [n_ex] * nvid)
    seq, pooled, layers = R.clipbert_base_model(ids, rep, mask, sd, return_layers=True)
    logits_ref = R.mlp_head(pooled, sd)
    with torch.no_grad():
        _, pooled16, layers16 = R.clipbert_base_model(ids, rep.detach(), mask, sd0, return_layers=True, rnd=R.Rounding.bf16())
        out16 = R.video_text_retrieval(ids, rep.detach(), mask, sd0, rnd=R.Rounding.bf16())
    gc = gridt.to(dev).to(torch.bfloat16).requires_grad_(True)
    tr._capture = {}
    o = tr(ids.to(dev), gc, mask.to(dev), labels=labels.to(dev), sample_size=nvid, _repeat_counts=[n_ex] * nvid)
    cap, tr._capture = tr._capture, None
    out("== transformer forward (6 seq, L=41): relerr vs bf16-matched oracle | vs fp32 oracle")
    out("  %-10s %.3e | %.3e" % ("embeddings", relerr(cap["embeddings"], layers16[0]), relerr(cap["embeddings"], layers[0])))
    for i in range(12):
        out("  layer%-5d %.3e | %.3e" % (i, relerr(cap["layer%d" % i], layers16[i + 1]), relerr(cap["layer%d" % i], layers[i + 1])))
    out("  %-10s %.3e | %.3e" % ("pooled", relerr(cap["pooled"], pooled16), relerr(cap["pooled"], pooled)))
    out("  %-10s %.3e | %.3e" % ("logits", relerr(o["logits"], out16["logits"]), relerr(o["logits"], logits_ref)))
    out("  logits got", o["logits"].detach().cpu().flatten().tolist())
    out("  logits m16", out16["logits"].flatten().tolist())
    out("  logits f32", logits_ref.detach().flatten().tolist())
    hpat = R.Rounding(relu_masks={"transformer.classifier.relu": (cap["c1"] > 0).cpu()})
    R.retrieval_loss(R.mlp_head(pooled, sd, rnd=hpat), labels).mean().backward()
    model.zero_grad()
    o["loss"].mean().backward()
    out("== transformer backward: gradient relerr / cosine vs fp32 oracle autograd (run's classifier ReLU pattern)")
    out("  %-60s %.3e  %.6f" % ("d(grid)", relerr(gc.grad, gr.grad), cosine(gc.grad, gr.grad)))
    for name, p in tr.named_parameters():
        r = sd["transformer." + name].grad
        if r is None or float(r.abs().sum()) == 0:
            continue
        e, c = relerr(p.grad, r), cosine(p.grad, r)
        if ("layer." not in name) or (".layer.0." in name) or (".layer.11." in name) or e > 2e-2:
            out("  %-60s %.3e  %.6f" % (name, e, c))
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    with open(os.path.join(ROOT, "tool_out", "parity_report.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
