"""Generate tests/golden/adamw.pt from the REFERENCE's own optimizer class (src/optimization/adamw.py, imported where it
lies) and torch.nn.utils.clip_grad_norm_, exactly as src/tasks/run_video_retrieval.py:477-487 drives them. Run beside a
checkout of the reference (CLIPBERT_REFERENCE_ROOT)."""
import importlib.util
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.nn.utils import clip_grad_norm_  # noqa: E402


def reference_adamw():
    from oracle import ref_import
    spec = importlib.util.spec_from_file_location("ref_adamw", os.path.join(ref_import.REFERENCE_ROOT, "src", "optimization", "adamw.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.AdamW


def case(seed=5, steps=4):
    g = torch.Generator().manual_seed(seed)
    shapes = [(7, 33), (129,), (3, 5, 3, 3), (200, 17), (64,)]
    params = [torch.randn(*s, generator=g) * 0.05 for s in shapes]
    grads = [[torch.randn(*s, generator=g) * (0.3 if t % 2 else 3.0) for s in shapes] for t in range(steps)]
    groups = [dict(idx=[0, 3], lr=5e-5, weight_decay=1e-3), dict(idx=[1, 4], lr=5e-5, weight_decay=0.0),
              dict(idx=[2], lr=2.5e-4, weight_decay=1e-3)]
    return params, grads, groups


def main():
    warnings.simplefilter("ignore")
    AdamW = reference_adamw()
    params, grads, groups = case()
    out = {}
    for max_norm in (-1.0, 2.0):
        ps = [torch.nn.Parameter(p.clone()) for p in params]
        opt = AdamW([dict(params=[ps[i] for i in g["idx"]], lr=g["lr"], weight_decay=g["weight_decay"]) for g in groups],
                    lr=5e-5, betas=(0.9, 0.98))
        traj, norms = [], []
        for gs in grads:
            for p, g_ in zip(ps, gs):
                p.grad = g_.clone()
            if max_norm > 0:
                norms.append(clip_grad_norm_(ps, max_norm).detach().clone())
            opt.step()
            opt.zero_grad()
            traj.append([p.detach().clone() for p in ps])
        out["max_norm_%g" % max_norm] = dict(traj=traj, norms=norms)
    torch.save(dict(source="reference: src/optimization/adamw.py AdamW (lr per group, betas (0.9, 0.98), eps 1e-6, correct_bias) + "
                           "torch.nn.utils.clip_grad_norm_, driven as run_video_retrieval.py:477-487", seed=5, steps=4, runs=out),
               os.path.join(ROOT, "tests", "golden", "adamw.pt"))
    print("wrote tests/golden/adamw.pt")


if __name__ == "__main__":
    main()
