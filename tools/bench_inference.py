"""Config 5 of BASELINE.json (paragraph-retrieval inference: 16 clips x 1 frame per video, 512-token captions, 8 captions per
forward) on one H100 - a measurement tool for the next round, NOT the contract bench (bench.py measures the training step).

    python tools/bench_inference.py [--flash 0|1] [--clips 16] [--captions 8] [--txt_len 512] [--size 224] [--steps 10]

One step = inference_retrieval's inner loop for one video (src/tasks/run_video_retrieval.py:639-666): the grids of the video's
clips (CNN once, ClipBert.encode_clips) and ONE transformer pass over clips x captions sequences (forward_clips(grid=...)).
Prints clips/s and the split CNN / transformer; --flash 1 routes attention (L = 521) to the mma.sync online-softmax kernel.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--flash", type=int, default=0)
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--captions", type=int, default=8)
    ap.add_argument("--txt_len", type=int, default=512)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import clipbert_b200 as cb
    from clipbert_b200 import ops
    from clipbert_b200 import workload as synth
    from clipbert_b200.workload import make_cfg
    dev = torch.device("cuda", 0)
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="R-50-grid.yaml", transformer_cls=cb.ClipBertForVideoTextRetrieval)
    model.load_state_dict(synth.cnn_state_dict(42), strict=False)
    model = model.to(dev).eval()
    model.cnn.pixel_mean = (123.675, 116.28, 103.53)
    ops.set_attention_flash(args.flash)
    u8 = synth.synth_images(1, args.clips * args.frames, size=args.size, seed=42, as_uint8=True).to(dev)
    ids, mask = synth.synth_text(args.captions, args.txt_len, seed=42)
    ids, mask = ids.to(dev), mask.to(dev)
    mb = dict(text_input_ids=ids, text_input_mask=mask, n_examples_list=[args.captions])

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    with torch.no_grad():
        grid = model.encode_clips(u8, args.clips)
        ms_cnn = timed(lambda: model.encode_clips(u8, args.clips))
        ms_tf = timed(lambda: model.forward_clips(dict(mb), args.clips, grid=grid))
        ms_all = timed(lambda: model.forward_clips(dict(mb), args.clips, grid=model.encode_clips(u8, args.clips)))
    L = args.txt_len + (args.size // 64) ** 2
    print(json.dumps(dict(workload="config 5: %d clips x %d frame, %d captions x %d tokens (L = %d), inference" % (
        args.clips, args.frames, args.captions, args.txt_len, L), attention="mma.sync online softmax" if args.flash else "CUDA-core online softmax",
        ms_cnn=round(ms_cnn, 3), ms_transformer=round(ms_tf, 3), ms_step=round(ms_all, 3), clips_per_s=round(args.clips / ms_all * 1e3, 1),
        sequences_per_s=round(args.clips * args.captions / ms_all * 1e3, 1))))


if __name__ == "__main__":
    main()
