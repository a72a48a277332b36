"""Generate tests/golden/transformer_base_outputs.pt from the REFERENCE's own ClipBertBaseModel (run where the reference tree is).

src/modeling/modeling.py:ClipBertBaseModel imported read-only through oracle/ref_import.py, fp32, eval mode, with
output_hidden_states = output_attentions = True (transformers.py:421-461): the (sequence_output, pooled_output,
all_hidden_states, all_attentions) tuple. Two cases: L = 32 + 9 = 41 (224 px frames, 3 x 3 grid) and L = 20 + 49 = 69
(448 px frames, 7 x 7 grid), with padded captions. Stored: the inputs, pooled_output, slices of every hidden state plus
its per-layer mean / std (as tools/make_golden.py does for the retrieval head), and the attention probabilities of
layers 0, 6 and 11 for the first sequence and its first two heads - a few hundred KB in all.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import ref_import, synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "transformer_base_outputs.pt")
ATT_LAYERS = (0, 6, 11)
ATT_HEADS = 2


def case(model, nseq, lt, gh, T, seed):
    g = torch.Generator().manual_seed(seed)
    grid = (torch.randn(nseq, T, gh, gh, 768, generator=g).abs() * 2).to(torch.bfloat16).float()
    ids, mask = synth.synth_text(nseq, lt, seed=seed + 1)
    with torch.no_grad():
        seq, pooled, hidden, attn = model(ids, grid, mask)
    assert len(hidden) == 13 and len(attn) == 12
    return dict(ids=ids, mask=mask, grid=grid.to(torch.bfloat16), L=lt + gh * gh, pooled=pooled.clone(),
                hidden_slices=torch.stack([h[:, :2, :32] for h in hidden]).clone(),
                hidden_stats=torch.tensor([[float(h.mean()), float(h.std())] for h in hidden]),
                seq_slice=seq[:, :, :32].clone(),
                attn_layers=ATT_LAYERS, attentions=torch.stack([attn[i][:1, :ATT_HEADS] for i in ATT_LAYERS]).clone())


def main():
    assert ref_import.available(), "needs the reference tree (oracle/ref_import.py)"
    m = ref_import.load()
    sd = synth.full_state_dict(42)
    cfg = ref_import.bert_config(output_hidden_states=True, output_attentions=True)
    model = m.ClipBertBaseModel(cfg)
    sub = {k[len("transformer.bert."):]: v for k, v in sd.items() if k.startswith("transformer.bert.")}
    missing, unexpected = model.load_state_dict(sub, strict=False)
    assert not [k for k in missing if "position_ids" not in k] and not unexpected, (missing, unexpected)
    model.eval()
    torch.save(dict(source="reference: src/modeling/modeling.py ClipBertBaseModel (imported via oracle/ref_import.py), fp32, eval, "
                           "output_hidden_states = output_attentions = True",
                    weights_seed=42, L41=case(model, 2, 32, 3, 2, 31), L69=case(model, 2, 20, 7, 1, 33)), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
