"""Module hooks, tensor hooks and torch.autograd.grad on GridFeatBackbone's stem, block, stage and grid-encoder outputs.

A hook on a module of feature.backbone or grid_encoder makes forward() run the modules (GridFeatBackbone._module_forward), so
torch's hook machinery applies to them as on the reference's detectron2 backbone. Checked here:
  cb_nhwc_intake                 bit-exact against a torch restatement (x.to(bf16), then (act > 0) ? v : +0) on every dtype and
                                 layout path, compact and zero-bordered outputs between NaN guard bands, > 2^31 elements;
  cb_unsubsample2_mask(act=NULL) bit-exact against its restatement;
  the module path                forward-hook outputs and the gradients tensor hooks see against the oracle's fp32 autograd
                                 along the run's own ReLU patterns; requires_grad of every output against d2's rule; observe-only
                                 hooks leave every parameter and frame gradient bit-identical to the default path; interventions
                                 (a gradient-rewriting tensor hook, forward-hook and pre-hook replacements) against the oracle
                                 with the same intervention; autograd semantics, memory and refusals.
tests/test_cnn_hooks_emulated.py replays the model-level runners below on a CPU with the emulated ops.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from model_util import cnn_patterns
from util import TOL_GRAD, relerr

BF16 = torch.bfloat16
STAGES = (("res2", 3, 1), ("res3", 4, 2), ("res4", 6, 2), ("res5", 3, 2))
BLOCKS = ["%s.%d" % (s, b) for s, nb, _ in STAGES for b in range(nb)]
SITES = (["feature.backbone", "feature.backbone.stem"] + ["feature.backbone." + s for s, _, _ in STAGES]
         + ["feature.backbone." + b for b in BLOCKS] + ["grid_encoder.0", "grid_encoder"])
TOL_FWD = 2e-2          # bf16 activations of a 50-conv stack against fp32 along the same ReLU patterns


@contextlib.contextmanager
def deterministic(on=True):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(on))
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


# ------------------------------------------------------------------------------------------------ cb_nhwc_intake restatement
def intake_ref(x, out, act=None, out_bordered=False, act_bordered=False):
    """The header's cb_nhwc_intake: one rounding to bf16, then (act > 0) ? v : +0, into the compact or bordered interior."""
    n, c, h, w = x.shape
    v = x.to(BF16).permute(0, 2, 3, 1)
    if act is not None:
        a = act.view(n, h + 2, w + 2, c)[:, 1:-1, 1:-1] if act_bordered else act.view(n, h, w, c)
        v = torch.where(a > 0, v, torch.zeros((), dtype=BF16, device=v.device))
    (out.view(n, h + 2, w + 2, c)[:, 1:-1, 1:-1] if out_bordered else out.view(n, h, w, c)).copy_(v)


def unsubsample2_ref(dsub, act, dx, n, h, w, c):
    """cb_unsubsample2_mask with act = NULL: dsub at even pixels, +0 elsewhere."""
    full = torch.zeros(n, h, w, c, dtype=BF16, device=dx.device)
    full[:, ::2, ::2] = dsub.view(n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c)
    dx.view(-1).copy_(full.reshape(-1))


def _source(layout, dtype, n, c, h, w, dev, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(n, c + 8, h + 1, w + 3, generator=g)
    base[0, 0, 0, :2] = float("nan")
    base[0, 1, 0, :2] = -0.0
    base = base.to(dtype).to(dev)
    if layout == "channels_last":
        return base[:, :c, :h, :w].contiguous(memory_format=torch.channels_last)
    if layout == "nchw":
        return base[:, :c, :h, :w].contiguous()
    if layout == "sliced_cl":          # channels-last, sliced: 8-aligned strides, 16-byte aligned start
        return base.permute(0, 2, 3, 1).contiguous()[:, 1:h + 1, 3:w + 3, 8:c + 8].permute(0, 3, 1, 2)
    if layout == "permuted":            # (n, h, c, w) storage
        return base[:, :c, :h, :w].permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)
    if layout == "sliced":
        return base[:, 3:c + 3, 1:h + 1, :w]
    if layout == "expanded":
        return base[:1, :c, :h, :w].expand(n, c, h, w)
    raise ValueError(layout)


def run_intake_case(dev, layout, dtype, bordered, mask, n=2, c=40, h=9, w=13, seed=0, impl=None):
    """One cb_nhwc_intake launch between NaN guard bands against intake_ref; returns None or raises AssertionError."""
    from clipbert_b200 import ops
    impl = impl or ops.nhwc_intake
    x = _source(layout, dtype, n, c, h, w, dev, seed)
    rows = n * (h + 2) * (w + 2) if bordered else n * h * w
    act = None
    if mask:
        g = torch.Generator().manual_seed(seed + 1)
        a = torch.randn(rows, c, generator=g)
        a[a.abs() < 0.3] = 0.0
        a[:3, :3] = float("nan")
        act = a.to(BF16).to(dev)
    guard = 64
    buf = torch.full((rows * c + 2 * guard,), float("nan"), dtype=BF16, device=dev)
    out = buf[guard: guard + rows * c].view(rows, c)
    if bordered:
        out.view(n, h + 2, w + 2, c).zero_()
        out.view(n, h + 2, w + 2, c)[:, 1:-1, 1:-1] = float("nan")       # interior poisoned, border must stay zero
    impl(x, out, act=act, out_bordered=bordered, act_bordered=bordered)
    want = out.clone()
    intake_ref(x, want, act=act, out_bordered=bordered, act_bordered=bordered)
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[-guard:]).all(), "guard band written"
    got, ref = out.float(), want.float()
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), "NaN positions differ"
    ok = ~torch.isnan(ref)
    assert torch.equal(bits(out)[ok.cpu()], bits(want)[ok.cpu()]), "values differ"
    if bordered:
        v = out.view(n, h + 2, w + 2, c)
        border = torch.ones(h + 2, w + 2, dtype=torch.bool, device=dev)
        border[1:-1, 1:-1] = False
        assert (bits(v[:, border]) == 0).all(), "border written"


INTAKE_LAYOUTS = ["channels_last", "nchw", "sliced_cl", "permuted", "sliced", "expanded"]
INTAKE_DTYPES = [torch.float32, BF16, torch.float16]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", INTAKE_LAYOUTS)
@pytest.mark.parametrize("dtype", INTAKE_DTYPES, ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("bordered", [False, True], ids=["compact", "bordered"])
@pytest.mark.parametrize("mask", [False, True], ids=["nomask", "mask"])
def test_nhwc_intake_elementwise(cuda, layout, dtype, bordered, mask):
    run_intake_case(cuda, layout, dtype, bordered, mask)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 8, 1, 1), (3, 2048, 7, 7), (2, 64, 65, 3), (1, 24, 130, 67)])
def test_nhwc_intake_shapes(cuda, shape):
    n, c, h, w = shape
    for layout in ("channels_last", "nchw", "sliced"):
        run_intake_case(cuda, layout, torch.float32, False, True, n=n, c=c, h=h, w=w, seed=c)
        run_intake_case(cuda, layout, BF16, True, False, n=n, c=c, h=h, w=w, seed=h)


@pytest.mark.gpu
def test_nhwc_intake_over_2_31_elements(cuda):
    """2^31 + 2^21 elements (bf16, channels-last, 4.3 GB each way): every element lands where it belongs."""
    from clipbert_b200 import ops
    n, c, h, w = 1, 2048, 1024, 1024 + 1
    x = torch.empty(n, h, w, c, dtype=BF16, device=cuda)
    x.view(h * w, c).copy_(torch.arange(c, device=cuda, dtype=torch.float32).to(BF16).expand(h * w, c))
    x[0, -1, -1, :] = 7.0
    out = torch.empty(n * h * w, c, dtype=BF16, device=cuda)
    assert x.numel() > 2 ** 31
    ops.nhwc_intake(x.permute(0, 3, 1, 2), out)
    assert torch.equal(out[:1], x.view(h * w, c)[:1]) and bool((out[-1] == 7.0).all())
    for r0 in range(0, h * w, 1 << 18):
        assert torch.equal(out[r0: r0 + (1 << 18)], x.view(h * w, c)[r0: r0 + (1 << 18)]), r0
    del x, out
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_nhwc_intake_rejects_bad_arguments(cuda):
    from clipbert_b200 import ops
    n0 = ops.launch_count()
    x = torch.randn(1, 12, 4, 4, device=cuda)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.nhwc_intake(x, torch.empty(16, 12, dtype=BF16, device=cuda))
    with pytest.raises(TypeError):
        ops.nhwc_intake(x.double()[:, :8], torch.empty(16, 8, dtype=BF16, device=cuda))
    out = torch.empty(16 * 8 + 1, dtype=BF16, device=cuda)[1:].view(16, 8)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.nhwc_intake(x[:, :8], out)
    from clipbert_b200.ops import _call
    with pytest.raises(RuntimeError, match="in_dtype"):
        _call("cb_nhwc_intake", x.data_ptr(), 1, 128, 16, 4, 1, 1, 8, 4, 4, None, 0, torch.empty(16, 8, dtype=BF16, device=cuda).data_ptr(), 0, None)
    with pytest.raises(RuntimeError, match="bad arguments"):
        _call("cb_nhwc_intake", None, 0, 128, 16, 4, 1, 1, 8, 4, 4, None, 0, None, 0, None)
    assert ops.launch_count() == n0


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 7, 7, 64), (1, 14, 13, 256), (3, 56, 56, 512)])
def test_unsubsample2_mask_free_elementwise(cuda, shape):
    from clipbert_b200 import ops
    n, h, w, c = shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    dsub = torch.randn(n * ho * wo, c, device=cuda).to(BF16)
    dsub[0, :4] = float("nan")
    dx = torch.full((n * h * w, c), float("nan"), dtype=BF16, device=cuda)
    want = torch.empty_like(dx)
    ops.unsubsample2_mask(dsub, None, dx, n, h, w, c)
    unsubsample2_ref(dsub, None, want, n, h, w, c)
    assert torch.equal(bits(dx), bits(want))


# ------------------------------------------------------------------------------------------------ model-level runners
def backbone(dev, sd, freeze_at=2):
    import clipbert_b200 as cb
    m = cb.GridFeatBackbone(freeze_at=freeze_at)
    assert not m.load_state_dict(sd).missing_keys
    return m.to(dev)


def sites(m):
    named = dict(m.named_modules())
    return [(s, named[s]) for s in SITES]


def observe(m, names=SITES):
    """Forward hooks on the named modules storing each output and, on outputs that require grad, a tensor hook storing the
    gradient it sees. Returns (store, handles)."""
    store = dict(out={}, grad={}, rg={})
    handles = []
    named = dict(m.named_modules())
    for name in names:
        def fh(mod, inp, out, name=name):
            t = out["res5"] if isinstance(out, dict) else out
            store["out"][name] = t
            store["rg"][name] = t.requires_grad
            if t.requires_grad:
                t.register_hook(lambda g, name=name: store["grad"].__setitem__(name, g))
        handles.append(named[name].register_forward_hook(fh))
    return store, handles


def frames(dev, size, n_frms=2, seed=5):
    from oracle import synth
    return synth.synth_images(1, n_frms, size=size, seed=seed).to(dev)


def run_patterns(m, x):
    """The ReLU patterns and pool selections of the default path's forward on x (its forward bits are the module path's)."""
    import test_gpu_input_grads as IG
    m._capture = {}
    with torch.enable_grad():
        grid = m(x.clone().requires_grad_(True))
    stash = m._capture["stash"]
    m._capture = None
    pat = cnn_patterns(stash, grid)
    return pat, IG.stem_patterns(stash), grid.detach()


def oracle(x, sd, pat, stem_pat, replace=None, grad_hooks=None):
    """The oracle's GridFeatBackbone (fp32, nothing detached) along the run's patterns, with every module output recorded and
    retaining its gradient. replace: {site: fn(output) -> new output}; grad_hooks: {site: tensor hook}."""
    import test_gpu_input_grads as IG
    from oracle import clipbert_ref as R
    outs = {}
    p = "cnn.feature.backbone."

    def rec(name, t):
        if replace and name in replace:
            t = replace[name](t)
        t.retain_grad()
        if grad_hooks and name in grad_hooks:
            t.register_hook(grad_hooks[name])
        outs[name] = t
        return t
    n, t_, c, h, w = x.shape
    with IG.oracle_stem(*stem_pat):
        y = rec("feature.backbone.stem", R.basic_stem(x.reshape(n * t_, c, h, w)[:, [2, 1, 0]], sd, p + "stem.", pat))
    for name, nb, stride in STAGES:
        for b in range(nb):
            y = rec("feature.backbone.%s.%d" % (name, b), R.bottleneck_block(y, sd, "%s%s.%d." % (p, name, b), stride if b == 0 else 1,
                                                                              b == 0, pat))
        outs["feature.backbone." + name] = y
    outs["feature.backbone"] = y
    g = rec("grid_encoder.0", F.conv2d(y, sd["cnn.grid_encoder.0.weight"], None, stride=1, padding=1))
    nn_, cc = g.shape[:2]
    g = g.flatten(2).gather(2, pat.pool_indices.flatten(2)).view(nn_, cc, g.shape[2] // 2, g.shape[3] // 2)
    g = rec("grid_encoder", pat.relu(g, "cnn.grid_encoder"))
    return g, outs


def required(name, freeze_at, frames_grad):
    """d2's rule: an output requires grad iff the frames do or a parameter at or below its module does."""
    if name.startswith("grid_encoder"):
        return True
    stage = name.split(".")[2] if name.count(".") >= 2 else "res5"
    if stage == "stem":
        return frames_grad
    return frames_grad or freeze_at <= [s for s, _, _ in STAGES].index(stage) + 1


def run_against_oracle(dev, sd, size, freeze_at, frames_grad, tol_fwd=TOL_FWD, tol_grad=TOL_GRAD):
    """Forward-hook outputs of every site and the gradients tensor hooks see at those that require grad, against the oracle."""
    m = backbone(dev, sd, freeze_at)
    x = frames(dev, size)
    pat, stem_pat, _ = run_patterns(m, x)
    store, handles = observe(m)
    xg = x.clone().requires_grad_(frames_grad)
    grid = m(xg)
    dgrid = torch.randn(grid.shape, generator=torch.Generator().manual_seed(size)).to(BF16)
    grid.backward(dgrid.to(dev))
    for hd in handles:
        hd.remove()
    leaf = x.detach().cpu().float().requires_grad_(True)
    with torch.enable_grad():
        ref, outs = oracle(leaf, sd, pat, stem_pat)
        ref.backward(dgrid.float().view(-1, *grid.shape[2:]).permute(0, 3, 1, 2))
    for name in SITES:
        assert store["rg"][name] == required(name, freeze_at, frames_grad), name
        e = relerr(store["out"][name], outs[name])
        assert e < tol_fwd, (name, e)
        if store["rg"][name]:
            e = relerr(store["grad"][name], outs[name].grad)
            assert e < tol_grad, (name, "grad", e)
    assert store["out"]["feature.backbone.res5"] is store["out"]["feature.backbone.res5.2"]
    if frames_grad:
        assert relerr(xg.grad, leaf.grad.view(xg.shape)) < tol_grad
    return store


def train_step(m, x, dgrid, hooks=False, frames_grad=True):
    """(grid, parameter gradients, frame gradient) of one backward, with or without observe-only hooks on every site."""
    for p in m.parameters():
        p.grad = None
    handles = observe(m)[1] if hooks else []
    xg = x.clone().requires_grad_(frames_grad)
    grid = m(xg)
    grid.backward(dgrid)
    for hd in handles:
        hd.remove()
    grads = {n: bits(p.grad) for n, p in m.named_parameters() if p.grad is not None}
    return bits(grid), grads, (bits(xg.grad) if frames_grad else None)


def run_observe_only_bits(dev, sd, size, freeze_at=2, frames_grad=True, runs=3):
    """Observe-only hooks: grid, every parameter gradient and the frame gradient bit-identical to the default path, run after run."""
    m = backbone(dev, sd, freeze_at)
    x = frames(dev, size)
    with deterministic():
        grid = m(x)
        dgrid = torch.randn(grid.shape, generator=torch.Generator().manual_seed(1)).to(BF16).to(dev)
        want = train_step(m, x, dgrid, frames_grad=frames_grad)
        for _ in range(runs):
            got = train_step(m, x, dgrid, hooks=True, frames_grad=frames_grad)
            assert torch.equal(got[0], want[0])
            assert got[1].keys() == want[1].keys() and all(torch.equal(got[1][k], want[1][k]) for k in want[1]), \
                [k for k in want[1] if not torch.equal(got[1][k], want[1][k])]
            if frames_grad:
                assert torch.equal(got[2], want[2])


def run_outputs_are_engine_activations(dev, sd, size):
    """Forward-hook outputs are the engine's own activations, bit for bit, as NCHW views."""
    m = backbone(dev, sd)
    x = frames(dev, size)
    m._capture = {}
    with torch.no_grad():
        m(x)
    cap = m._capture
    m._capture = None
    store, handles = observe(m)
    with torch.no_grad():
        m(x)
    for hd in handles:
        hd.remove()
    for b in BLOCKS:
        y = cap[b]["y"]
        out = store["out"]["feature.backbone." + b]
        n, c, h, w = out.shape
        ref = y.view(n, h + 2, w + 2, c)[:, 1:-1, 1:-1] if y.shape[0] != n * h * w else y.view(n, h, w, c)
        assert torch.equal(bits(out.permute(0, 2, 3, 1)), bits(ref)), b
        assert out.dtype == BF16 and out.permute(0, 2, 3, 1).is_contiguous() == (b != "res5.2")
    s = store["out"]["feature.backbone.stem"]
    assert torch.equal(bits(s.permute(0, 2, 3, 1)), bits(cap["stem"]))
    assert torch.equal(bits(store["out"]["grid_encoder.0"].permute(0, 2, 3, 1).reshape(-1, 768)), bits(cap["gconv"]))


def run_interventions(dev, sd, size):
    """A tensor hook zeroing channels of res4[3]'s gradient, a forward hook replacing res3[1]'s output with an fp32 NCHW tensor,
    and a pre-hook replacing res4[0]'s input, each against the oracle with the same intervention."""
    with deterministic():
        _run_interventions(dev, sd, size)


def _run_interventions(dev, sd, size):
    m = backbone(dev, sd)
    x = frames(dev, size)
    pat, stem_pat, _ = run_patterns(m, x)
    dgrid = torch.randn(1, 2, size // 64, size // 64, 768, generator=torch.Generator().manual_seed(2)).to(BF16)
    leaf = x.detach().cpu().float().requires_grad_(True)
    base = train_step(m, x, dgrid.to(dev))

    # (1) gradient rewrite
    def zero_ch(g):
        g = g.clone()
        g[:, :512] = 0
        return g
    store, handles = observe(m, ["feature.backbone.res4.2", "feature.backbone.stem"])
    hd = m.feature.backbone.res4[3].register_forward_hook(lambda mod, i, o: o.register_hook(zero_ch) and None)
    for p in m.parameters():
        p.grad = None
    xg = x.clone().requires_grad_(True)
    m(xg).backward(dgrid.to(dev))
    hd.remove()
    for h_ in handles:
        h_.remove()
    with torch.enable_grad():
        ref, outs = oracle(leaf, sd, pat, stem_pat, grad_hooks={"feature.backbone.res4.3": zero_ch})
        ref.backward(dgrid.float().view(-1, *dgrid.shape[2:]).permute(0, 3, 1, 2))
    assert relerr(store["grad"]["feature.backbone.res4.2"], outs["feature.backbone.res4.2"].grad) < TOL_GRAD
    assert relerr(xg.grad, leaf.grad.view(xg.shape)) < TOL_GRAD
    changed = {n for n, p in m.named_parameters() if p.grad is not None and not torch.equal(bits(p.grad), base[1][n])}
    assert {n for n in changed if ".res4.4." in n or ".res5." in n or "grid_encoder" in n} == set()
    assert any(".res4.0." in n for n in changed) and any(".res3." in n for n in changed)

    # (2) forward-hook replacements with fp32 NCHW (a block, and the res5 stage: taken into the zero-bordered layout),
    # (3) a pre-hook replacement with a bf16 channels-last tensor
    def half_fp32(t):
        return (t.float() * 0.5).contiguous()

    def scale_in(t):
        return t * 0.75
    for site, kind, fn in (("feature.backbone.res3.1", "fwd", half_fp32), ("feature.backbone.res5", "fwd", half_fp32),
                           ("feature.backbone.res4.0", "pre", scale_in)):
        mod = dict(m.named_modules())[site]
        m._capture = {}
        hd = (mod.register_forward_hook(lambda mod, i, o, fn=fn: fn(o)) if kind == "fwd"
              else mod.register_forward_pre_hook(lambda mod, i, fn=fn: (fn(i[0]),)))
        store, handles = observe(m, ["grid_encoder.0", "grid_encoder"] + ["feature.backbone." + b for b in BLOCKS])
        xg = x.clone().requires_grad_(True)
        grid = m(xg)
        grid.backward(dgrid.to(dev))
        hd.remove()
        for h_ in handles:
            h_.remove()
        pat2 = replay_patterns(m._capture, store, grid)
        m._capture = None
        prev = BLOCKS[BLOCKS.index(site.split(".", 2)[2]) - 1] if kind == "pre" else None
        rep = {"feature.backbone." + prev: fn} if kind == "pre" else {site + ".2" if site.endswith("res5") else site: fn}
        leaf.grad = None
        with torch.enable_grad():
            ref, outs = oracle(leaf, sd, pat2, stem_pat, replace=rep)
            ref.backward(dgrid.float().view(-1, *dgrid.shape[2:]).permute(0, 3, 1, 2))
        assert relerr(grid, ref.permute(0, 2, 3, 1).reshape(grid.shape)) < TOL_FWD, site
        assert relerr(xg.grad, leaf.grad.view(xg.shape)) < TOL_GRAD, site


def replay_patterns(cap, store, grid):
    """cnn_patterns of a module-path run from its _capture (block activations) and the hook-stored geometry."""
    blocks = []
    for b in BLOCKS:
        out = store["out"]["feature.backbone." + b]
        blocks.append(dict(name=b, h=out.shape[2], w=out.shape[3], a_pad=cap[b]["a_pad"], b=cap[b]["b"], y=cap[b]["y"]))
    g0 = store["out"]["grid_encoder.0"]
    n, c, h, w = g0.shape
    stash = dict(n=n, h=h, w=w, blocks=blocks, gconv=g0.detach().permute(0, 2, 3, 1).reshape(-1, c))
    return cnn_patterns(stash, grid)


def run_semantics(dev, sd, size):
    """autograd.grad leaves the flat gradient buffer untouched, backward() accumulates, retain_graph allows a second backward and
    its absence gives torch's error, stored outputs survive the next forward, no_grad / inference_mode feature extraction."""
    m = backbone(dev, sd)
    x = frames(dev, size)
    store, handles = observe(m, ["feature.backbone.res5.2", "feature.backbone.res4.5"])
    grid = m(x)
    m._flat.grad.fill_(float("nan"))
    before = bits(m._flat.grad)
    res5 = store["out"]["feature.backbone.res5.2"]
    g, = torch.autograd.grad(grid.float().sum(), res5, retain_graph=True)
    assert torch.equal(bits(m._flat.grad), before)
    assert relerr(g, store["grad"]["feature.backbone.res5.2"]) == 0
    m._flat.grad.zero_()
    grid.float().sum().backward(retain_graph=True)
    once = m._flat.grad.clone()
    assert float(once.abs().sum()) > 0
    grid.float().sum().backward()
    assert relerr(m._flat.grad, once * 2) < 1e-6        # accumulated (the weight-gradient sums add into the buffer in fp32)
    with pytest.raises(RuntimeError, match="backward through the graph a second time"):
        grid.float().sum().backward()
    # backward(inputs=...) with an output: that output's .grad, no parameter gradient
    grid = m(x)
    m._flat.grad.zero_()
    r4 = store["out"]["feature.backbone.res4.5"]
    grid.float().sum().backward(inputs=[r4])
    assert r4.grad is not None and float(m._flat.grad.abs().sum()) == 0
    for hd in handles:
        hd.remove()
    # stored outputs are not overwritten by the next forward; no_grad and inference_mode agree with the default path
    store, handles = observe(m, ["feature.backbone.res5.2"])
    with torch.no_grad():
        m(x)
    kept = store["out"]["feature.backbone.res5.2"]
    snap = kept.clone()
    with torch.no_grad():
        m(frames(dev, size, seed=9))
    assert torch.equal(kept, snap)
    with torch.inference_mode():
        a = m(x)
    for hd in handles:
        hd.remove()
    with torch.no_grad():
        b = m(x)
    assert torch.equal(bits(a), bits(b))


def run_refusals(dev, sd):
    m = backbone(dev, sd)
    x = frames(dev, 64, n_frms=1)
    bb = m.feature.backbone
    for mod, what in ((bb.res3[0].conv1, "feature.backbone.res3.0.conv1"), (bb.stem.conv1.norm, "feature.backbone.stem.conv1.norm")):
        hd = mod.register_forward_hook(lambda *a: None)
        with pytest.raises(RuntimeError, match=what.replace(".", r"\.")):
            m(x)
        hd.remove()
    for mod in (bb, bb.stem):
        hd = mod.register_forward_pre_hook(lambda *a: None)
        with pytest.raises(RuntimeError, match="pre-hooks"):
            m(x)
        hd.remove()
    with pytest.raises(RuntimeError, match="runs only inside GridFeatBackbone.forward"):
        bb(x[0])
    hd = bb.res5[2].register_forward_hook(lambda *a: None)
    m._bucket_hook = lambda *a: None
    with pytest.raises(RuntimeError, match="enable_overlapped_allreduce"):
        m(x)
    m._bucket_hook = None
    hd.remove()
    m(x)           # nothing left behind


@pytest.fixture(scope="module")
def cnn_sd():
    from oracle import synth
    return synth.cnn_state_dict(42)


@pytest.mark.gpu
@pytest.mark.parametrize("size,freeze_at,frames_grad", [(224, 2, True), (224, 2, False), (224, 1, False), (224, 3, True),
                                                         (224, 3, False), (448, 2, True)])
def test_hook_outputs_and_gradients_match_oracle(cuda, cnn_sd, size, freeze_at, frames_grad):
    run_against_oracle(cuda, cnn_sd, size, freeze_at, frames_grad)


@pytest.mark.gpu
@pytest.mark.parametrize("freeze_at,frames_grad", [(2, True), (2, False), (1, False), (3, True)])
def test_observe_only_hooks_leave_gradients_bit_identical(cuda, cnn_sd, freeze_at, frames_grad):
    run_observe_only_bits(cuda, cnn_sd, 224, freeze_at, frames_grad)


@pytest.mark.gpu
def test_hook_outputs_are_the_engine_activations(cuda, cnn_sd):
    run_outputs_are_engine_activations(cuda, cnn_sd, 224)


@pytest.mark.gpu
def test_interventions_match_oracle(cuda, cnn_sd):
    run_interventions(cuda, cnn_sd, 224)


@pytest.mark.gpu
def test_autograd_semantics(cuda, cnn_sd):
    run_semantics(cuda, cnn_sd, 224)


@pytest.mark.gpu
def test_refusals(cuda, cnn_sd):
    run_refusals(cuda, cnn_sd)


@pytest.mark.gpu
def test_memory_returns_to_baseline(cuda, cnn_sd):
    m = backbone(cuda, cnn_sd)
    x = frames(cuda, 224)
    store, handles = observe(m)
    m(x.clone().requires_grad_(True)).float().sum().backward()       # warm the pools
    store["out"].clear(), store["grad"].clear()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    grid = m(x.clone().requires_grad_(True))
    assert torch.cuda.memory_allocated() > base
    grid.float().sum().backward()
    del grid
    store["out"].clear(), store["grad"].clear()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == base
    for hd in handles:
        hd.remove()


@pytest.mark.gpu
def test_no_hooks_same_launches(cuda, cnn_sd):
    from clipbert_b200 import ops
    m = backbone(cuda, cnn_sd)
    x = frames(cuda, 224)

    def count():
        n0 = ops.launch_count()
        m(x).float().sum().backward()
        torch.cuda.synchronize()
        return ops.launch_count() - n0
    count()
    a = count()
    hd = m.feature.backbone.res4[3].register_forward_hook(lambda *a: None)
    count()
    hd.remove()
    assert count() == a


@pytest.mark.gpu
def test_grad_cam_and_layer_cam_match_oracle(cuda, cnn_sd):
    """pytorch-grad-cam's recipe written out (forward hook + tensor hook on res5[-1]), LayerCAM on res4, and
    register_full_backward_hook on a block, on a score of the grid, against the oracle's CAMs."""
    m = backbone(cuda, cnn_sd)
    x = frames(cuda, 224)
    pat, stem_pat, _ = run_patterns(m, x)
    acts, grads, bwd = {}, {}, {}

    def keep(name):
        def fh(mod, i, o):
            acts[name] = o
            o.register_hook(lambda g: grads.__setitem__(name, g))
        return fh
    hs = [m.feature.backbone.res5[-1].register_forward_hook(keep("res5")), m.feature.backbone.res4.register_forward_hook(keep("res4")),
          m.feature.backbone.res4[2].register_full_backward_hook(lambda mod, gi, go: bwd.__setitem__("res4.2", (gi[0], go[0])))]
    grid = m(x)
    w = torch.randn(768, generator=torch.Generator().manual_seed(4)).to(cuda)
    (grid.float() * w).sum().backward()
    for h_ in hs:
        h_.remove()
    gradcam = F.relu((grads["res5"].float().mean((2, 3), keepdim=True) * acts["res5"].float()).sum(1))
    layercam = F.relu((F.relu(grads["res4"].float()) * acts["res4"].float()).sum(1))
    leaf = x.detach().cpu().float().requires_grad_(True)
    with torch.enable_grad():
        ref, outs = oracle(leaf, cnn_sd, pat, stem_pat)
        (ref.permute(0, 2, 3, 1) * w.cpu()).sum().backward()
    r5, r4 = outs["feature.backbone.res5.2"], outs["feature.backbone.res4.5"]
    assert relerr(gradcam, F.relu((r5.grad.mean((2, 3), keepdim=True) * r5).sum(1))) < TOL_GRAD
    assert relerr(layercam, F.relu((F.relu(r4.grad) * r4).sum(1))) < TOL_GRAD
    gi, go = bwd["res4.2"]
    assert relerr(go, outs["feature.backbone.res4.2"].grad) < TOL_GRAD and relerr(gi, outs["feature.backbone.res4.1"].grad) < TOL_GRAD
