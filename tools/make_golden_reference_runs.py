"""Generate tests/golden/reference_runs.pt: outputs of the reference's OWN code (transformer classes, AdamW, the two checkpoint
helpers of src/utils/load_save.py, the optimizer grouping of src/optimization/utils.py, get_resize_size of src/datasets/data_utils.py) on the inputs of the tests that compare
against them - tests/test_oracle.py, tests/test_load_save.py, tests/test_host_logic.py - so that those comparisons run without the reference tree. Needs the reference checkout
(CLIPBERT_REFERENCE_ROOT); the vocabulary-wide masked-LM scores are stored as a slice, their arg-max and their log-sum-exp."""
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import ref_import, synth  # noqa: E402

MLM_SLICE = 256       # vocabulary columns of the masked-LM scores stored verbatim


def checksums(sd):
    """key -> (shape, float64 sum, float64 sum of squares, the first 16 values): enough to pin a tensor without storing it"""
    out = {}
    for k, v in sd.items():
        v = torch.as_tensor(v)
        f = v.detach().double().flatten()
        out[k] = (tuple(v.shape), float(f.sum()), float((f * f).sum()), f[:16].float().clone())
    return out


def transformer_runs(weights):
    g = torch.Generator().manual_seed(123)
    grid = torch.randn(3, 2, 3, 3, 768, generator=g).abs()
    ids, mask = synth.synth_text(3, 20, seed=77)
    labels = torch.tensor([0, 1, 1])
    with torch.no_grad():
        ref = ref_import.build_reference_transformer(weights)(ids, grid, mask, labels=labels)
    out = dict(retrieval=dict(logits=ref["logits"].clone(), loss=ref["loss"].clone()))
    sd = dict(weights)
    sd.update(synth.transformer_state_dict(51, num_labels=3129))
    tgt = (torch.rand(3, 3129, generator=g) > 0.99).float()
    with torch.no_grad():
        ref = ref_import.build_reference_transformer(sd, "ClipBertForSequenceClassification", num_labels=3129, loss_type="bce")(
            ids, grid, mask, labels=tgt)
    out["sequence_classification"] = dict(logits=ref["logits"].clone(), loss=ref["loss"].clone())
    # pre-training with train-mode random sampling of 7 of 20 visual tokens, numpy seed 1234
    sd = {k: v for k, v in weights.items() if not k.startswith("transformer.classifier.")}
    sd.update({k: v for k, v in synth.transformer_state_dict(60, head="pretraining").items() if k.startswith("transformer.cls.")})
    g = torch.Generator().manual_seed(5)
    grid = torch.randn(2, 2, 4, 5, 768, generator=g).abs()
    ids, mask = synth.synth_text(2, 12, seed=9)
    model = ref_import.build_reference_transformer(sd, "ClipBertForPreTraining", hidden_dropout_prob=0.0,
                                                   attention_probs_dropout_prob=0.0, pixel_random_sampling_size=7)
    model.train()
    np.random.seed(1234)
    with torch.no_grad():
        ref = model(ids, grid, mask)
    model.eval()
    with torch.no_grad():
        ref_eval = model(ids, grid, mask)
    mlm = ref["mlm_scores"]
    out["pretraining_sampled"] = dict(itm_scores=ref["itm_scores"].clone(), mlm_slice=mlm[..., :MLM_SLICE].clone(),
                                      mlm_argmax=mlm.argmax(-1), mlm_logsumexp=torch.logsumexp(mlm.double(), -1).float(),
                                      itm_scores_eval=ref_eval["itm_scores"].clone())
    return out


def adamw_run():
    import make_golden_adamw as mk      # noqa: E402  (tools/)
    AdamW = mk.reference_adamw()
    params, grads, groups = mk.case(seed=21, steps=3)
    ps = [torch.nn.Parameter(p.clone()) for p in params]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt = AdamW([dict(params=[ps[i] for i in g["idx"]], lr=g["lr"], weight_decay=g["weight_decay"]) for g in groups], lr=1e-4)
        for gs in grads:
            for p, g_ in zip(ps, gs):
                p.grad = g_.clone()
            opt.step()
    return dict(seed=21, steps=3, params=[p.detach().clone() for p in ps])


def load_save_runs(tmp):
    import test_load_save as T
    ref = T._reference_functions()
    tv = T._tv_resnet50_state_dict()
    path = os.path.join(tmp, "tv.pth")
    torch.save(tv, path)
    conv = ref["convert_torchvision_ckpt_to_detectron2"](path)
    sd = {k[len("transformer."):]: v for k, v in synth.full_state_dict(7).items() if k.startswith("transformer.")}
    sd["classifier.2.weight"] = torch.zeros(7, 1536)
    sd["extra.weight"] = torch.zeros(3)
    a = T._model().transformer
    ref["load_state_dict_with_mismatch"](a, sd)
    return dict(convert_keys=list(conv["model"].keys()), convert_heuristics=conv["matching_heuristics"],
                convert_checksums=checksums(conv["model"]), mismatch_checksums=checksums(a.state_dict()))


def optimizer_groups():
    """The reference's own setup_e2e_optimizer (src/optimization/utils.py:96-161) on THIS package's ClipBert: the parameter names
    of each of its eight groups, with their lr / weight decay."""
    import types
    import clipbert_b200 as cb
    from util import make_cfg
    sys.path.insert(0, ref_import.REFERENCE_ROOT)
    from src.optimization.utils import setup_e2e_optimizer
    model = cb.ClipBert(make_cfg(), detectron2_model_cfg="R-50-grid.yaml", transformer_cls=cb.ClipBertForVideoTextRetrieval)
    opts = types.SimpleNamespace(learning_rate=5e-5, weight_decay=1e-3, transformer_lr_mul=1.0, transformer_lr_mul_prefix="",
                                 cnn_learning_rate=5e-5, cnn_weight_decay=1e-3, cnn_lr_mul=1.0, cnn_lr_mul_prefix="grid_encoder",
                                 optim="adamw", betas=(0.9, 0.98))
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(names=[names[id(p)] for p in g["params"]], lr=g["lr"], weight_decay=g["weight_decay"])
            for g in setup_e2e_optimizer(model, opts).param_groups]


RESIZE_CASES = [(360, 640, 448), (640, 360, 448), (224, 224, 224), (37, 53, 96), (1080, 1920, 768), (500, 499, 1000)]


def resize_sizes():
    """get_resize_size for tensors (src/datasets/data_utils.py:166-198) on RESIZE_CASES: (h, w, size) -> (new_h, new_w)"""
    import ast
    ref_path = os.path.join(ref_import.REFERENCE_ROOT, "src", "datasets", "data_utils.py")
    tree = ast.parse(open(ref_path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "get_resize_size"]
    ns = {"torch": torch}
    exec(compile(ast.Module(body=fn, type_ignores=[]), ref_path, "exec"), ns)
    return {(h, w, s): tuple(int(v) for v in ns["get_resize_size"](torch.zeros(3, h, w), s)) for h, w, s in RESIZE_CASES}


def main():
    import tempfile
    assert ref_import.available(), "reference tree not found at %s (set CLIPBERT_REFERENCE_ROOT)" % ref_import.REFERENCE_ROOT
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    weights = synth.full_state_dict(42)
    out = dict(source="the reference's own src/modeling/modeling.py classes, src/optimization/adamw.py AdamW and "
                      "src/utils/load_save.py helpers and src/optimization/utils.py setup_e2e_optimizer, run by tools/make_golden_reference_runs.py")
    out.update(transformer_runs(weights))
    out["adamw"] = adamw_run()
    out["optimizer_groups"] = optimizer_groups()
    out["resize_sizes"] = resize_sizes()
    with tempfile.TemporaryDirectory() as tmp:
        out["load_save"] = load_save_runs(tmp)
    dst = os.path.join(ROOT, "tests", "golden", "reference_runs.pt")
    torch.save(out, dst)
    print("wrote %s (%d bytes)" % (dst, os.path.getsize(dst)))


if __name__ == "__main__":
    main()
