"""Generate tests/golden/wra.npz by running the UNMODIFIED reference's ITM word-region alignment code
(data/itm.py, model/ot.py, model/pretrain.py) on CPU:

    python tests/golden/make_wra_goldens.py          # needs a reference checkout ($UNITER_REFERENCE)

* `batch/*`: itm_ot_collate on seeded samples (`wra_samples`), every field including `ot_inputs`;
* `ot/*`: optimal_transport_dist in float64 on seeded 16-bit-representable rows (`ot_inputs_f64`), its
  values and the gradients of its text and image inputs for seeded upstream gradients;
* `itm/*`: a tiny UniterForPretraining (weights: synth.seeded_state(schema, WRA_STATE_SEED), checksum
  stored) in fp32, eval mode: the ITM forward with ot_inputs on the `batch` samples at D = 64, its
  itm_loss, ot_pos, ot_neg, the pre-training loss with itm_ot_lambda 0.1 (pretrain.py:272-290) and the
  gradients of a few parameters.

Torch 2.x rejects the reference's uint8 masks in masked_fill_ / masked_select, so the pads are passed as
bool and model/ot.py's `trace` is replaced by the diagonal sum; nothing else is changed.  The reference is
imported through the shims of make_goldens.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_goldens import import_reference, import_reference_data, state_checksum  # noqa: E402

WRA_STATE_SEED = 21
ITM_OT_LAMBDA = 0.1
GRAD_KEYS = ("itm_output.weight", "uniter.pooler.dense.weight", "uniter.img_embeddings.img_linear.weight",
             "uniter.encoder.layer.0.attention.self.query.weight")


def trace_diag(x):
    return torch.diagonal(x, dim1=1, dim2=2).sum(-1)


def wra_samples(seed, n, D=16):
    """Per-pair tuples as ItmDataset.__getitem__ returns them (data/itm.py:80-93), seeded; includes a pair
    with one region and one with one text token."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        tl = 1 if i == 2 else int(torch.randint(2, 10, (1,), generator=g))
        nbb = 1 if i == 1 else int(torch.randint(2, 9, (1,), generator=g))
        ids = torch.randint(1000, 1999, (tl,), generator=g)
        feat, pos = torch.randn(nbb, D, generator=g), torch.rand(nbb, 7, generator=g)
        am = torch.ones(tl + nbb, dtype=torch.long)
        out.append((ids, feat, pos, am, torch.tensor([int(i % 3 != 0)])))
    return out


def ot_inputs_f64(seed, B=5, D=48):
    """Padded float64 text / image rows (values representable in fp16) with bool pads, and upstream
    gradients of the distances."""
    g = torch.Generator().manual_seed(seed)
    tl = [int(v) for v in torch.randint(1, 12, (B,), generator=g)]
    nb = [int(v) for v in torch.randint(1, 15, (B,), generator=g)]
    M, N = max(tl), max(nb)
    txt = (torch.randn(B, M, D, generator=g) + 0.3).half().double()
    img = (torch.randn(B, N, D, generator=g) - 0.2).half().double()
    txt_pad = torch.arange(M)[None, :] >= torch.tensor(tl)[:, None]
    img_pad = torch.arange(N)[None, :] >= torch.tensor(nb)[:, None]
    txt, img = txt.masked_fill(txt_pad[..., None], 0), img.masked_fill(img_pad[..., None], 0)
    return txt, img, txt_pad, img_pad, torch.randn(B, generator=g).double()


def run_wra(out_path):
    rm, _, rpre = import_reference()
    import_reference_data()
    import data.itm as ritm
    import model.ot as rot
    from uniter_b200.synth import seeded_state
    rot.trace = trace_diag
    rec = {}
    batch = ritm.itm_ot_collate(wra_samples(81, 6))
    for k, v in batch.items():
        if k == "ot_inputs":
            for kk, vv in v.items():
                rec["batch/ot_inputs/" + kk] = vv.numpy() if torch.is_tensor(vv) else np.array(vv)
        else:
            rec["batch/" + k] = v.numpy()
    for case, seed in (("a", 5), ("b", 6)):
        txt, img, tp, ip, g = ot_inputs_f64(seed)
        txt.requires_grad_(True)
        img.requires_grad_(True)
        dist = rot.optimal_transport_dist(txt, img, tp, ip)
        dist.backward(g)
        for k, v in (("txt", txt.detach()), ("img", img.detach()), ("txt_pad", tp), ("img_pad", ip), ("g", g),
                     ("dist", dist.detach()), ("d_txt", txt.grad), ("d_img", img.grad)):
            rec["ot/%s/%s" % (case, k)] = v.numpy()
    cfg = rm.UniterConfig(2000, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
                          max_position_embeddings=64, type_vocab_size=2)
    model = rpre.UniterForPretraining(cfg, 64, 11)
    st = seeded_state({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=WRA_STATE_SEED)
    model.load_state_dict(st, strict=True)
    model.eval()
    b = ritm.itm_ot_collate(wra_samples(81, 6, D=64))
    b["ot_inputs"] = dict(b["ot_inputs"], txt_pad=b["ot_inputs"]["txt_pad"].bool(),
                          img_pad=b["ot_inputs"]["img_pad"].bool())
    itm_loss, (ot_pos, ot_neg) = model(b, task="itm", compute_loss=True)
    loss = itm_loss.mean() + ITM_OT_LAMBDA * (ot_pos.sum() - ot_neg.sum()) / (ot_pos.size(0) + ot_neg.size(0))
    loss.backward()
    rec["itm/checksum"] = np.array(state_checksum(st))
    rec["itm/itm_loss"] = itm_loss.detach().numpy()
    rec["itm/ot_pos"] = ot_pos.detach().numpy()
    rec["itm/ot_neg"] = ot_neg.detach().numpy()
    rec["itm/loss"] = loss.detach().numpy()
    params = dict(model.named_parameters())
    for k in GRAD_KEYS:
        rec["itm/grad/" + k] = params[k].grad.numpy()
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path, "%.1f KB" % (os.path.getsize(out_path) / 1024))


if __name__ == "__main__":
    run_wra(os.path.join(HERE, "wra.npz"))
