"""Cost of the deterministic mode (torch.use_deterministic_algorithms(True)) on two training steps: the headline step (bench.py's
default configuration) and the 448 px MSRVTT step (`tools/profile_step.py --size 448 --txt_len 20 --n_ex 2 --n_clips 8
--batch 16`). A step is forward_clips + the fused clip-LSE loss + backward + FusedAdamW (gradient-norm clip and update), eager.

Three modes alternate in one session: flag off; flag on with torch's NaN fill of uninitialised memory (its default); flag on
without the fill (torch.utils.deterministic.fill_uninitialized_memory = False), which separates the cost of the fill from that
of the kernels. Step times are CUDA events over `--steps` steps, in `--rounds` alternating rounds. Then one step per mode runs
with an event pair around every launch, and the device time of the launches the mode changes is listed per entry point.
Prints, and writes tool_out/deterministic.txt. Usage: python tools/profile_deterministic.py [--steps 10 --rounds 3]"""
import argparse
import os
import subprocess
import sys
import types
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import bench  # noqa: E402

WORKLOADS = {
    "headline 224 px": dict(batch=32, n_clips=2, n_frm=2, size=224, txt_len=32, n_ex=1),
    "MSRVTT 448 px": dict(batch=16, n_clips=8, n_frm=2, size=448, txt_len=20, n_ex=2),
}
MODES = ("off", "on + NaN fill", "on, no fill")


def _family(label):
    """the entry points whose launches the mode changes (None: unchanged)"""
    if label.startswith("gemm mode=1") or label.startswith("gemm wgrad group"):
        return "wgrad GEMM (single + grouped)"
    for k in ("cb_layernorm_bwd", "cb_embed_text_bwd", "cb_embed_visual_bwd", "cb_colsum", "cb_sumsq", "cb_clip_lse_loss"):
        if label.startswith(k):
            return k
    return None


def _mode(name):
    torch.use_deterministic_algorithms(name != "off")
    torch.utils.deterministic.fill_uninitialized_memory = name != "on, no fill"


def run_workload(name, w, steps, rounds):
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from clipbert_b200 import workload as synth
    from clipbert_b200.optim import FusedAdamW
    from clipbert_b200.workload import make_cfg
    dev = torch.device("cuda:0")
    torch.manual_seed(42)
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="x")
    model.load_state_dict(synth.cnn_state_dict(42), strict=False)
    model = model.to(dev).train()
    model.cnn.pixel_mean = bench.IMAGE_MEAN
    opt = FusedAdamW([p for p in model.parameters() if p.requires_grad], lr=1e-5, model=model)
    args = types.SimpleNamespace(head="retrieval", **w)
    d = {k: v.to(dev) for k, v in bench.make_host_batch(args, 0).items()}
    mb = dict(visual_inputs=d["visual_inputs"], text_input_ids=d["text_input_ids"], text_input_mask=d["text_input_mask"],
              labels=d["labels"], n_examples_list=[w["n_ex"]] * w["batch"])

    def step():
        model.zero_grad()
        logits = model.forward_clips(dict(mb), w["n_clips"])["logits"]
        cb.clip_lse_loss(logits, d["labels"]).backward()
        opt.clip_grad_norm(1.0)
        opt.step()

    times = defaultdict(list)
    for mode in MODES:                       # warm every mode's shapes (workspaces, split plans, module loads)
        _mode(mode)
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for mode in MODES:
            _mode(mode)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            times[mode].append(e0.elapsed_time(e1) / steps)
    per_launch = {}
    for mode in MODES:
        _mode(mode)
        ev = []
        ops.set_op_timing(ev)
        step()
        torch.cuda.synchronize()
        ops.set_op_timing(None)
        agg = defaultdict(lambda: [0.0, 0])
        for label, a, b in ev:
            fam = _family(label)
            if fam is not None:
                agg[fam][0] += a.elapsed_time(b)
                agg[fam][1] += 1
        per_launch[mode] = agg
    _mode("off")
    torch.utils.deterministic.fill_uninitialized_memory = True
    lines = ["== %s (batch %d, %d clips x %d frames, %d px, %d tokens, %d captions per video)" % (
        name, w["batch"], w["n_clips"], w["n_frm"], w["size"], w["txt_len"], w["n_ex"])]
    base = min(times["off"])
    for mode in MODES:
        t = times[mode]
        lines.append("  step, flag %-14s min %8.2f ms  max %8.2f ms  (%+.1f %% vs off, min to min)" % (mode, min(t), max(t), 100 * (min(t) / base - 1)))
    lines.append("  device time per step of the launches the mode changes (ms, launches; the plain cb_sumsq is not bracketed):")
    fams = sorted({f for m in MODES for f in per_launch[m]})
    lines.append("    %-32s" % "" + "".join("%24s" % m for m in MODES))
    for f in fams:
        lines.append("    %-32s" % f + "".join("%16.3f ms x%-4d" % tuple(per_launch[m].get(f, [0.0, 0])) for m in MODES))
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default="tool_out/deterministic.txt")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    lines = ["card: %s (name, power limit, max SM clock)" % card]
    for name in args.workloads.split(","):
        lines += run_workload(name, WORKLOADS[name], args.steps, args.rounds)
        print("\n".join(lines), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    open(args.out, "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
