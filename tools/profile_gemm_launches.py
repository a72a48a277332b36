"""Device time of every GEMM shape of one training step, each timed on its own: the cb_gemm descriptors of one eager step are
recorded (as bench.py's roofline pass does), then every distinct descriptor is replayed --reps times back to back on one stream
between CUDA events. Unlike tools/profile_step.py, no host gap and no side-stream kernel lands inside a launch's window. The tile
column is the tile the launch ran with (128 x 256 on TN / NN: both consumer warpgroups on one tile). --ab also times every TN / NN
shape forced onto 128 x 256 tiles and kept off them (cb_gemm_desc.reserved CB_GEMM_FORCE_WIDE / CB_GEMM_NO_WIDE).
Writes tool_out/gemm_launches.txt (or --out). Usage: python tools/profile_gemm_launches.py [--reps 20] [--ab]"""
import argparse
import os
import sys
from collections import OrderedDict

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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ab", action="store_true")
    ap.add_argument("--out", default="tool_out/gemm_launches.txt")
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
    B = args.batch

    def step():
        model.zero_grad()
        mb = dict(visual_inputs=d["visual_inputs"], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"],
                  labels=d["labels"], n_examples_list=[args.n_ex] * B)
        logits = model.forward_clips(mb, args.n_clips)["logits"]
        cb.clip_lse_loss(logits, d["labels"]).backward()

    ops.set_pdl(0)
    ops.overlap_wgrad = False
    for _ in range(2):
        step()
    ops._gemm_record = []
    step()
    torch.cuda.synchronize()
    rec, ops._gemm_record = ops._gemm_record, None
    shapes = OrderedDict()
    for kw in rec:
        if "group" in kw:
            continue
        shapes.setdefault(ops.gemm_key(kw), [kw, 0])[1] += 1
    peaks = bench.load_peaks()
    rows = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def time_us(kw):
        for _ in range(3):
            ops.gemm(**kw)
        e0.record()
        for _ in range(args.reps):
            ops.gemm(**kw)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.reps

    for key, (kw, cnt) in shapes.items():
        us = time_us(kw)
        tile = "128x%d" % ops.gemm_tile_width(kw)
        ab = ""
        if args.ab and kw.get("mode", 0) != ops.CB_GEMM_WGRAD:
            ab = " %9.1f %9.1f" % (time_us(dict(kw, reserved=ops.GEMM_NO_WIDE)), time_us(dict(kw, reserved=ops.GEMM_FORCE_WIDE)))
        fl = 2.0 * kw["m"] * kw["n"] * kw["k"] * kw.get("ntaps", 1)
        by = bench.gemm_algorithmic_bytes(kw)
        ideal = max(fl / (peaks["tflops"] * 1e12), by / (peaks["hbm"] * 1e9)) * 1e6
        rows.append((us * cnt / 1e3, key, cnt, us, ideal, "hbm" if by / (peaks["hbm"] * 1e9) > fl / (peaks["tflops"] * 1e12) else "tensor",
                     tile, ab))
    lines = ["GEMM launches of one step (grouped wgrad launches excluded), each shape replayed %d x back to back; ideal = max(flop / %.0f"
             " TF/s, algorithmic bytes / %.0f GB/s)" % (args.reps, peaks["tflops"], peaks["hbm"]),
             "%-62s %4s %9s %9s %9s %6s %6s %8s" % ("shape", "n", "us", "ms/step", "ideal us", "frac", "bound", "tile")
             + (" %9s %9s" % ("us <=128", "us 256") if args.ab else "")]
    for ms, key, cnt, us, ideal, bound, tile, ab in sorted(rows, key=lambda r: -r[0]):
        lines.append("%-62s %4d %9.1f %9.3f %9.1f %6.2f %6s %8s" % (key, cnt, us, ms, ideal, ideal / us, bound, tile) + ab)
    lines.append("total %.3f ms/step over %d launches" % (sum(r[0] for r in rows), sum(r[2] for r in rows)))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    open(args.out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
