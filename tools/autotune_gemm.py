"""Measure the launch configuration of every distinct GEMM of the training step on the GPU it runs on.

Records the cb_gemm descriptors of one fwd+bwd step of the bench workload, then for each distinct shape times the candidate
(tile width, wgrad K-split, k-chunks per stage) inside a CUDA graph and writes the winners to
clipbert_b200/gemm_tuning.json, which ops.gemm consults at run time ("measure, don't guess"). The table is meant to be
committed with the GPU model it was measured on (its "device" field); the per-shape report goes to tool_out/.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import bench  # noqa: E402


def record_step(args):
    """cb_gemm descriptors of ONE step of the bench workload ``args`` describes (bench.CONFIGS: train steps and config 5's inference)."""
    import clipbert_b200 as cb
    from clipbert_b200 import ops, workload as synth
    from clipbert_b200.workload import make_cfg
    if not hasattr(args, "head") or args.head is None:
        args.config = getattr(args, "config", "headline")
        bench.apply_config(args)
    dev = torch.device("cuda:0")
    torch.manual_seed(42)
    if args.head == "multiple_choice":
        model = cb.ClipBert(make_cfg(num_labels=args.n_ex), detectron2_model_cfg="x", transformer_cls=cb.ClipBertForMultipleChoice)
    else:
        model = cb.ClipBert(make_cfg(), detectron2_model_cfg="x")
    model.load_state_dict(synth.cnn_state_dict(42), strict=False)
    model = model.to(dev)
    model = model.eval() if args.inference else model.train()
    model.cnn.pixel_mean = bench.IMAGE_MEAN
    host = bench.make_host_batch(args, 0)
    d = {k: v.to(dev) for k, v in host.items()}
    B, n_clips, T, n_ex = args.batch, args.n_clips, args.n_frm, args.n_ex
    os.environ["CB_NO_TUNING"] = "1"
    ops._tuning = {}
    ops._gemm_record = []
    if args.inference:
        with torch.no_grad():
            grid = model.encode_clips(d["visual_inputs"], n_clips)
            model.forward_clips(dict(text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"], n_examples_list=[n_ex] * B), n_clips, grid=grid)
    else:
        if getattr(args, "clip_batching", 1):
            mb = dict(visual_inputs=d["visual_inputs"], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"], n_examples_list=[n_ex] * B)
            if args.head == "retrieval":
                mb["labels"] = d["labels"]
            logits = model.forward_clips(mb, n_clips)["logits"]
        else:
            vis = d["visual_inputs"].view(B, n_clips, T, 3, args.size, args.size)
            logits = []
            for c in range(n_clips):
                mb = dict(visual_inputs=vis[:, c], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"],
                          labels=d["labels"] if args.head == "retrieval" else None, n_examples_list=[n_ex] * B)
                logits.append(model(mb)["logits"])
        bench.lse_loss(logits, d["labels"]).backward()
    torch.cuda.synchronize()
    rec, ops._gemm_record = ops._gemm_record, None
    return rec


def synth_call(kw, dev):
    """Fresh random operands of the recorded shapes (the tuner must not depend on the step's live tensors)."""
    def rnd(r, c):
        return (torch.randn(r, c, device=dev) * 0.1).to(torch.bfloat16)
    out = dict((k, v) for k, v in kw.items() if not isinstance(v, torch.Tensor))
    mode, m, n, k, taps = kw.get("mode", 0), kw["m"], kw["n"], kw["k"], kw.get("ntaps", 1)
    a_rows, a_ld, b_rows, b_ld = kw["a_rows"], kw["a_ld"], kw["b_rows"], kw["b_ld"]
    out["a"] = rnd(a_rows + 4, a_ld)[:a_rows]
    out["b"] = rnd(b_rows, b_ld)
    if mode == 1:
        out["out"] = torch.zeros(m, kw["out_ld"], device=dev)
        if kw.get("scale") is not None:
            out["scale"] = torch.rand(m, device=dev) + 0.5
    else:
        rowmap = kw.get("rowmap", 0)
        if rowmap == 1:
            h, w = kw["map_h"], kw["map_w"]
            rows = (m // (h * w)) * (h + 2) * (w + 2)
        else:
            rows = m
        dt = torch.float32 if kw.get("out_fp32") else torch.bfloat16
        out["out"] = torch.zeros(rows, kw["out_ld"], device=dev, dtype=dt)
        for name, ldk in (("residual", "res_ld"), ("aux", "aux_ld")):
            if kw.get(name) is not None:
                out[name] = rnd(m, kw[ldk])
        if kw.get("out2") is not None:
            out["out2"] = torch.zeros(rows, kw["out2_ld"], device=dev, dtype=torch.bfloat16)
        for name in ("scale", "shift"):
            if kw.get(name) is not None:
                out[name] = torch.rand(n, device=dev) + 0.5
    return out


def time_cfg(ops, call, reps=10):
    try:
        ops.gemm(**call)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                for _ in range(reps):
                    ops.gemm(**call)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
        return best
    except RuntimeError:
        torch.cuda.synchronize()
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="headline", choices=sorted(bench.CONFIGS))
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--n_clips", type=int, default=None)
    ap.add_argument("--n_frm", type=int, default=None)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--txt_len", type=int, default=None)
    ap.add_argument("--n_ex", type=int, default=None)
    ap.add_argument("--head", default=None)
    ap.add_argument("--inference", type=int, default=None)
    ap.add_argument("--clip_batching", type=int, default=1)
    ap.add_argument("--out", default=os.path.join(ROOT, "clipbert_b200", "gemm_tuning.json"))
    ap.add_argument("--merge", type=int, default=1)
    args = bench.apply_config(ap.parse_args())
    from clipbert_b200 import ops
    dev = torch.device("cuda:0")
    t0 = time.time()
    rec = record_step(args)
    uniq = {}
    counts = {}
    rec = [m for kw in rec for m in (kw["group"] if "group" in kw else [kw])]      # grouped wgrads: tune / list their members
    for kw in rec:
        key = ops.gemm_key(kw)
        uniq.setdefault(key, kw)
        counts[key] = counts.get(key, 0) + 1
    print("recorded %d GEMM launches, %d distinct shapes (%.1f s)" % (len(rec), len(uniq), time.time() - t0), flush=True)
    del rec
    torch.cuda.empty_cache()
    table, report = {}, []
    saved = 0.0
    for key, kw in uniq.items():
        call = synth_call(kw, dev)
        base = time_cfg(ops, call)
        cands = []
        n, mode = kw["n"], kw.get("mode", 0)
        bns = [b for b in (64, 128, 256) if b <= max(64, n) or b == 64]
        if mode == 1:
            kc = -(-kw["k"] // 64)
            for bn in bns:
                for sp in sorted(set(x for x in (1, 2, 3, 4, 6, 8, 12, 16, 24) if x <= kc)):
                    cands.append((bn, sp, 0))
        else:
            for bn in bns:
                for kch in (0, 1, 2, 4):
                    cands.append((bn, 0, kch))
        # two CTAs per SM (reserved bit 5): 128 x 64 tiles only
        cands = [c + (0,) for c in cands] + [c + (1,) for c in cands if c[0] == 64 and c[2] in (0, 1)]
        best, best_t = None, base if base is not None else 1e9
        for (bn, sp, kch, occ2) in cands:
            reserved = (kch << 8) | (32 if occ2 else 64)
            if bn == 256 and mode != 1:      # TN / NN 128 x 256 tiles are forced through reserved (block_n = 256 means 128 there)
                reserved |= ops.GEMM_FORCE_WIDE
            t = time_cfg(ops, dict(call, block_n=0 if reserved & ops.GEMM_FORCE_WIDE else bn, split_k=sp, reserved=reserved))
            if t is not None and t < best_t * 0.97:
                best, best_t = (bn, sp, kch, occ2), t
        if best is not None:
            table[key] = list(best)
            saved += (base - best_t) * counts[key] if base is not None else 0.0
        report.append("%-58s x%-3d model %7.2f us  best %7.2f us  %s" % (key, counts[key], base if base else -1, best_t, best))
        print(report[-1], flush=True)
        del call
    old = {}
    if args.merge and os.path.exists(args.out):
        try:
            old = json.load(open(args.out)).get("configs", {})
        except Exception:
            old = {}
    old.update(table)
    json.dump(dict(device=torch.cuda.get_device_name(0), note="(block_n, split_k, kch, two CTAs per SM) per GEMM shape (TN / NN block_n 256: "
                   "the 128 x 256 tile); see tools/autotune_gemm.py",
                   configs=old), open(args.out, "w"), indent=0, sort_keys=True)
    print("tuned %d / %d shapes; predicted saving %.2f ms per step; wrote %s (%.1f s)" % (len(table), len(uniq), saved / 1e3, args.out, time.time() - t0))
    os.makedirs(os.path.join(ROOT, "tool_out"), exist_ok=True)
    open(os.path.join(ROOT, "tool_out", "autotune_report_%s.txt" % args.config), "w").write("\n".join(report) + "\n")


if __name__ == "__main__":
    main()
