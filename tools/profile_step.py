"""Per-kernel device-time breakdown of one training step (eager launches, CUDA events around every launch).
Writes tool_out/step_breakdown.txt. Usage: python tools/profile_step.py [--batch 32 --n_clips 2 ...]"""
import argparse
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--n_clips", type=int, default=2)
    ap.add_argument("--n_frm", type=int, default=2)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--txt_len", type=int, default=32)
    ap.add_argument("--n_ex", type=int, default=1)
    ap.add_argument("--clip_batching", type=int, default=1)
    ap.add_argument("--out", default="tool_out/step_breakdown.txt")
    ap.add_argument("--ncu", type=int, default=0, help="1: bracket ONE step with cudaProfilerStart/Stop for "
                    "`ncu --profile-from-start off` instead of timing with events")
    args = ap.parse_args()
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from clipbert_b200 import workload as synth
    from clipbert_b200.workload import make_cfg
    dev = torch.device("cuda:0")
    torch.manual_seed(42)
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="x")
    model.load_state_dict(synth.cnn_state_dict(42), strict=False)
    model = model.to(dev).train()
    model.cnn.pixel_mean = bench.IMAGE_MEAN
    host = bench.make_host_batch(args, 0)
    d = {k: v.to(dev) for k, v in host.items()}
    B, n_clips, T, n_ex = args.batch, args.n_clips, args.n_frm, args.n_ex

    ops.set_pdl(0)      # per-launch durations: no prologue/tail overlap between consecutive kernels

    def step():
        model.zero_grad()
        if args.clip_batching:
            mb = dict(visual_inputs=d["visual_inputs"], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"],
                      labels=d["labels"], n_examples_list=[n_ex] * B)
            logits = model.forward_clips(mb, n_clips)["logits"]
        else:
            vis = d["visual_inputs"].view(B, n_clips, T, 3, args.size, args.size)
            logits = []
            for c in range(n_clips):
                mb = dict(visual_inputs=vis[:, c], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"],
                          labels=d["labels"], n_examples_list=[n_ex] * B)
                logits.append(model(mb)["logits"])
        cb.clip_lse_loss(logits, d["labels"]).backward()          # the fused clip-LSE loss, as bench.py runs it

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    if args.ncu:
        torch.cuda.profiler.start()
        step()
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        return
    ev = []
    ops.set_op_timing(ev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    step()
    e1.record()
    torch.cuda.synchronize()
    ops.set_op_timing(None)
    total = e0.elapsed_time(e1)
    agg = defaultdict(lambda: [0.0, 0])
    for label, a, b in ev:
        agg[label][0] += a.elapsed_time(b)
        agg[label][1] += 1
    ksum = sum(v[0] for v in agg.values())
    lines = ["step %.3f ms (eager, with event overhead); sum of kernel times %.3f ms; %d launches" % (total, ksum, len(ev))]
    fam = defaultdict(float)
    for label, (ms, cnt) in agg.items():
        fam[label.split(" ")[0] + (" " + label.split(" ")[1] if label.startswith("gemm") else "")] += ms
    lines.append("-- by family")
    for k, v in sorted(fam.items(), key=lambda kv: -kv[1]):
        lines.append("  %-28s %8.3f ms  %5.1f %%" % (k, v, 100 * v / ksum))
    peaks = bench.load_peaks()
    lines.append("-- by kernel/shape: total ms, count, avg us; for gemm: TFLOP/s, algorithmic GB/s (A + B + out + residual + aux, each once),"
                 " ideal us = max(flop/%.0f TF/s, bytes/%.0f GB/s), lost ms = total - count x ideal" % (peaks["tflops"], peaks["hbm"]))
    rows = []
    for label, (ms, cnt) in agg.items():
        tf, lost = "", 0.0
        if label.startswith("gemm mode="):     # ("gemm wgrad group xN": several problems in one launch, no single shape)
            f = dict(kv.split("=") for kv in label.split(" ")[1:])
            m, n, k, taps, mode = int(f["m"]), int(f["n"]), int(f["k"]), int(f["taps"]), int(f["mode"])
            fl = 2.0 * m * n * k * taps
            if mode == 1:      # wgrad: A = dY [k, m], B = X [k, n], out fp32 [m, taps*n] (red.add: read + write)
                by = 2.0 * k * (m + n) + 8.0 * m * n * taps
            else:
                by = 2.0 * m * k + 2.0 * n * k * taps + (4.0 if f.get("f32") == "1" else 2.0) * m * n * (1 + int(f.get("o2", 0))) \
                    + 2.0 * m * n * (int(f.get("res", 0)) + int(f.get("aux", 0)))
            us = 1e3 * ms / cnt
            ideal = max(fl / (peaks["tflops"] * 1e12), by / (peaks["hbm"] * 1e9)) * 1e6
            lost = (us - ideal) * cnt / 1e3
            tf = "%7.1f TF/s %7.0f GB/s  ideal %6.1f us  lost %6.3f ms" % (fl / us / 1e6, by / us / 1e3, ideal, lost)
        rows.append((lost if label.startswith("gemm mode=") else ms, label, ms, cnt, tf))
    for _, label, ms, cnt, tf in sorted(rows, key=lambda r: -r[2]):
        lines.append("  %-62s %8.3f ms x%-4d %8.1f us %s" % (label, ms, cnt, 1e3 * ms / cnt, tf))
    lines.append("-- gemm shapes by lost time")
    for lost, label, ms, cnt, tf in sorted((r for r in rows if r[1].startswith("gemm mode=")), key=lambda r: -r[0])[:25]:
        lines.append("  %-62s lost %6.3f ms of %6.3f" % (label, lost, ms))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    open(args.out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:60]))


if __name__ == "__main__":
    main()
