"""Activation recomputation (GridFeatBackbone.recompute_activations + ClipBertBaseModel.recompute_activations): peak memory and
step time of an eager ClipBert retrieval training step (forward_clips, clip_lse_loss, backward; dropout 0.1, FREEZE_AT 2) with
both switches off and both on, at the headline configuration (32 videos x 2 clips x 2 frames, 224 px, 1 caption), at MSRVTT's
448 px sampling (16 videos x 8 clips x 2 frames, 2 captions) and at denser samplings of the same videos: 16 clips x 2 frames,
and 28 clips x 2 frames, which needs the switches to fit on an 80 GB card.

Per setting and mode: torch.cuda.max_memory_allocated over one step after two warm-up steps, on a model built fresh for that
mode (nothing left over from the other mode: the CNN's pool of zero-bordered buffers only grows), and the step time from CUDA
events around each eager step, on one model, `--rounds` rounds of `--steps` steps with the two modes alternating round by round;
the median and the spread (min - max of the round medians). A mode that runs out of memory is reported as such. The card name, power limit and max
SM clock are read in the same run.
Usage: python tools/profile_recompute.py [--rounds 5 --steps 3 --out tool_out/recompute.txt]"""
import argparse
import gc
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from profile_input_grads import card  # noqa: E402

SETTINGS = [("headline", 32, 2, 2, 224, 1), ("MSRVTT 448 px", 16, 8, 2, 448, 2), ("denser", 16, 16, 2, 448, 2), ("denser", 16, 28, 2, 448, 2)]


_WEIGHTS = []


def build():
    import clipbert_b200 as cb
    from oracle import synth
    from util import make_cfg
    if not _WEIGHTS:
        _WEIGHTS.append(synth.full_state_dict(42))
    model = cb.ClipBert(make_cfg(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1), detectron2_model_cfg="R-50-grid.yaml")
    model.load_state_dict(_WEIGHTS[0])
    return model.to(torch.device("cuda:0")).train()


def set_mode(model, on):
    model.cnn.recompute_activations = on
    model.transformer.bert.recompute_activations = on


def release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def setting(out, name, videos, clips, frames, size, n_ex, rounds, steps):
    import clipbert_b200 as cb
    from oracle import synth
    dev = torch.device("cuda:0")
    batch = synth.synth_batch(videos, clips * frames, n_ex=n_ex, size=size, seed=1)
    mb = {k: (v.to(dev) if torch.is_tensor(v) else list(v)) for k, v in batch.items()}
    labels = mb.pop("labels")
    model = None

    def step():
        model.zero_grad()
        logits = model.forward_clips(dict(mb), clips)["logits"]
        cb.clip_lse_loss(logits, labels).backward()

    peak, times = {}, {False: [], True: []}
    for on in (False, True):
        model = build()
        set_mode(model, on)
        try:
            for _ in range(2):
                step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            step()
            torch.cuda.synchronize()
            peak[on] = torch.cuda.max_memory_allocated() / 2 ** 30
        except torch.OutOfMemoryError:
            peak[on] = None
        model = None
        release()
    model = build()
    for _ in range(rounds):
        for on in (False, True):
            if peak[on] is None:
                continue
            set_mode(model, on)
            e = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
            e[0].record()
            for k in range(steps):
                step()
                e[k + 1].record()
            torch.cuda.synchronize()
            times[on].append(statistics.median(e[k].elapsed_time(e[k + 1]) for k in range(steps)))
    what = "%s: %d videos x %d clips x %d frames, %d px, %d caption(s)" % (name, videos, clips, frames, size, n_ex)
    for on in (False, True):
        mode = "on " if on else "off"
        if peak[on] is None:
            out("%-70s switches %s  out of memory" % (what, mode))
            continue
        t = times[on]
        out("%-70s switches %s  max_memory_allocated %6.2f GiB  step %8.2f ms (rounds %.2f - %.2f)" % (
            what, mode, peak[on], statistics.median(t), min(t), max(t)))
    model = None
    del mb, batch
    release()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_recompute.py measures on the GPU"
    lines = []

    def out(s):
        print(s, flush=True)
        lines.append(s)
    out(card())
    for s in SETTINGS:
        setting(out, *s, args.rounds, args.steps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
