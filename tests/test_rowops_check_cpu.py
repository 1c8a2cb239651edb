"""CPU: the checker of tests/rowops_check.py.  It must accept a float32 stand-in for a kernel result
and reject each single-item mutation of it that a masking, scaling, row-selection or accumulation bug
would produce."""
import copy

import pytest
import torch

from oracle import philox
from tests import rowops_check as rc

ROWS, H, SEED, STREAM = 37, 264, 17, (5 << 20) | 4


def test_keep_mask_indexes_row_times_ncols():
    keep, inv = rc.keep_mask(SEED, STREAM, 0.3, 5, 24, counter=3)
    thr, inv2 = philox.dropout_params(0.3)
    r, c = 3, 17
    assert inv == inv2
    assert bool(keep[r, c]) == bool(philox.rand16(SEED, STREAM + (3 << 20), r * 24 + c) >= thr)
    assert abs(keep.float().mean().item() - 0.7) < 0.1


def _ln_case(dtype, p, on_dy, row_kind, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(ROWS, H, generator=g) * 2 + 0.3).to(dtype)
    gamma = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype)
    dy = torch.randn(ROWS, H, generator=g).to(dtype)
    init = [torch.randn(H, generator=g) for _ in range(3)]
    kinds = torch.randint(0, 2, (ROWS,), generator=g, dtype=torch.int32) if row_kind else None
    keep, inv = rc.keep_mask(SEED, STREAM, p, ROWS, H) if p else (None, 1.0)
    dx0 = torch.randn(ROWS, H, generator=g).to(dtype) if row_kind else None
    kw = dict(keep=keep, inv_keep=inv, on_dy=on_dy, row_kind=kinds, kind=1, dx0=dx0,
              dgamma0=init[0], dbeta0=init[1], dbias0=init[2])
    ref = rc.ln_bwd_reference(dy, x, gamma, **kw)
    act = ref["active"]
    base = rc.ln_bwd_baseline(dy[act], x[act], gamma, keep[act] if keep is not None else None, inv, on_dy)
    f32 = rc.ln_bwd_reference(dy, x, gamma, dtype=torch.float32, **kw)
    good = dict(dx=f32["dx"].to(dtype), dx_drop=f32["dx_drop"].to(dtype) if f32["dx_drop"] is not None else None,
                dgamma=f32["dgamma"], dbeta=f32["dbeta"], dbias=f32["dbias"])
    return x, gamma, dy, init, kinds, keep, inv, dx0, ref, base, good


def _expect_fail(fails, name, what):
    assert any(f.startswith(name) for f in fails), "%s not caught in %s: %s" % (what, name, fails)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ln_bwd_checker_dropout_on_dx(dtype):
    x, gamma, dy, init, _, keep, inv, _, ref, base, good = _ln_case(dtype, 0.1, False, False)
    chk = dict(dgamma0=init[0], dbeta0=init[1], dbias0=init[2])
    assert not rc.check_ln_bwd(good, ref, base, dtype, **chk)

    def lin_mut(dx_drop):
        m = copy.deepcopy(good)
        m["dx_drop"] = dx_drop.to(dtype)
        m["dbias"] = init[2] + m["dx_drop"].float().sum(0)     # consistent with the mutated branch
        return rc.check_ln_bwd(m, ref, base, dtype, **chk)

    dx32 = good["dx"].float()
    shifted = torch.roll(keep.reshape(-1), 1).reshape(ROWS, H)
    _expect_fail(lin_mut(dx32 * shifted * inv), "dx_drop", "mask shifted by one element")
    _expect_fail(lin_mut(dx32 * keep), "dx_drop", "missing 1/keep scale")

    xh = (x.double() - x.double().mean(1, keepdim=True))
    xh = xh / torch.sqrt((xh ** 2).mean(1, keepdim=True) + rc.EPS)
    for r in (0, ROWS // 2):
        m = copy.deepcopy(good)                                   # one row missing from dgamma
        m["dgamma"] = good["dgamma"] - (dy[r].double() * xh[r]).float()
        _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dgamma", "row missing from dgamma")
        m = copy.deepcopy(good)                                   # ... from dbeta / dbias
        m["dbeta"] = good["dbeta"] - dy[r].float()
        m["dbias"] = good["dbias"] - good["dx_drop"][r].float()
        fails = rc.check_ln_bwd(m, ref, base, dtype, **chk)
        _expect_fail(fails, "dbeta", "row missing from dbeta")
        _expect_fail(fails, "dbias", "row missing from dbias")
    m = copy.deepcopy(good)                                       # initial value dropped
    m["dgamma"] = good["dgamma"] - init[0]
    _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dgamma", "initial dgamma ignored")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ln_bwd_checker_dropout_on_dy_with_row_kind(dtype):
    x, gamma, dy, init, kinds, keep, inv, dx0, ref, base, good = _ln_case(dtype, 0.1, True, True, seed=1)
    chk = dict(dx0=dx0, dgamma0=init[0], dbeta0=init[1], dbias0=init[2])
    assert not rc.check_ln_bwd(good, ref, base, dtype, **chk)
    act = ref["active"]
    r_in = int((~act).nonzero()[0])
    r_act = int(act.nonzero()[-1])

    m = copy.deepcopy(good)                                       # a touched inactive row
    m["dx"][r_in, 5] = 0
    _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dx (inactive rows)", "touched inactive row")
    m = copy.deepcopy(good)                                       # inactive rows zeroed
    m["dx"][~act] = 0
    _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dx (inactive rows)", "zeroed inactive rows")

    for what, kp, iv in (("mask shifted by one element", torch.roll(keep.reshape(-1), 1).reshape(ROWS, H), inv),
                         ("missing 1/keep scale", keep, 1.0)):
        f32 = rc.ln_bwd_reference(dy, x, gamma, keep=kp, inv_keep=iv, on_dy=True, row_kind=kinds, kind=1,
                                  dx0=dx0, dgamma0=init[0], dbeta0=init[1], dbias0=init[2], dtype=torch.float32)
        m = dict(dx=f32["dx"].to(dtype), dx_drop=None, dgamma=f32["dgamma"], dbeta=f32["dbeta"], dbias=f32["dbias"])
        fails = rc.check_ln_bwd(m, ref, base, dtype, **chk)
        for n in ("dx:", "dbeta"):
            _expect_fail(fails, n, what)

    m = copy.deepcopy(good)                                       # an inactive row counted in dbeta
    m["dbeta"] = good["dbeta"] + (dy[r_in].double() * keep[r_in] * inv).float()
    _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dbeta", "inactive row in dbeta")
    m = copy.deepcopy(good)                                       # an active row missing from dbeta
    m["dbeta"] = good["dbeta"] - (dy[r_act].double() * keep[r_act] * inv).float()
    _expect_fail(rc.check_ln_bwd(m, ref, base, dtype, **chk), "dbeta", "active row missing from dbeta")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ln_fwd_checker(dtype):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(ROWS, H, generator=g) * 2).to(dtype)
    x[::5] = (x[::5].float() + 100).to(dtype)                        # |mean| >> std
    gamma = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype)
    beta = (0.1 * torch.randn(H, generator=g)).to(dtype)
    ref = rc.ln_fwd_reference(x, gamma, beta)
    base = rc.ln_fwd_baseline(x, gamma, beta)
    good = rc.ln_fwd_reference(x, gamma, beta, torch.float32).to(dtype)
    assert not rc.check_rows("y", good, ref, base, dtype)[0]
    m = good.clone()
    m[3] = (good[3].float() - beta.float()).to(dtype)               # beta missing from one row
    _expect_fail(rc.check_rows("y", m, ref, base, dtype)[0], "y", "missing beta")
    # statistics of a row with |mean| >> std taken in 16 bits
    r = 5
    xr = x[r].float()
    mu16 = xr.mean().to(dtype).float()
    m = good.clone()
    m[r] = ((xr - mu16) / torch.sqrt(((xr - mu16) ** 2).mean() + rc.EPS) * gamma.float() + beta.float()).to(dtype)
    _expect_fail(rc.check_rows("y", m, ref, base, dtype)[0], "y", "16-bit mean of an offset row")


def _embed_case(dtype, seed=3):
    from uniter_b200.synth import seeded_state, uniter_state_shapes
    Hs, V, P, D = 64, 50, 20, 7
    state = {k: v for k, v in seeded_state(uniter_state_shapes(Hs, 0, 4, V, P, 2, D), seed=seed).items()
             if not k.startswith("pooler")}
    state = {k: v.to(dtype).float() for k, v in state.items()}       # the model's 16-bit weights
    g = torch.Generator().manual_seed(seed)
    T = 29
    rows = dict(kind=torch.randint(0, 2, (T,), generator=g), word_id=torch.randint(0, V, (T,), generator=g),
                pos_id=torch.randint(0, P, (T,), generator=g), type_id=torch.randint(0, 2, (T,), generator=g))
    rows["img_src"] = torch.where(rows["kind"] == 1, torch.randint(0, 40, (T,), generator=g), -1)
    G = torch.randn(T, Hs, generator=g).to(dtype)
    box = torch.rand(40, 7, generator=g).to(dtype)
    keep, inv = rc.keep_mask(SEED, STREAM, 0.1, T, Hs)
    ref = rc.embed_rows_reference(state, rows, G, box, keep, inv)
    base = rc.embed_rows_reference(state, rows, G, box, keep, inv, dtype=dtype)
    f32 = rc.embed_rows_reference(state, rows, G, box, keep, inv, dtype=torch.float32)
    return state, rows, G, box, keep, inv, ref, base, {k: v.to(dtype) for k, v in f32.items()}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_embed_rows_checker(dtype):
    state, rows, G, box, keep, inv, ref, base, good = _embed_case(dtype)
    for n in ("x", "u", "ppre"):
        fails, _ = rc.check_rows(n, good[n], ref[n], base[n], dtype)
        assert not fails, fails
    assert torch.equal(good["ppre"][rows["kind"] == 0], torch.zeros_like(good["ppre"][rows["kind"] == 0]))
    x0 = rc.embed_rows_reference(state, rows, G, box, dtype=torch.float32)["x"]
    T, Hs = G.shape
    for what, kp, iv in (("mask shifted by one element", torch.roll(keep.reshape(-1), 1).reshape(T, Hs), inv),
                         ("missing 1/keep scale", keep, 1.0)):
        m = (x0 * kp * iv).to(dtype)
        _expect_fail(rc.check_rows("x", m, ref["x"], base["x"], dtype)[0], "x", what)
    t_img = int((rows["kind"] == 1).nonzero()[0])                     # one image row given its text twin's type
    rows2 = dict(rows, type_id=rows["type_id"].clone())
    rows2["type_id"][t_img] = 1 - rows2["type_id"][t_img]
    m = rc.embed_rows_reference(state, rows2, G, box, keep, inv, dtype=torch.float32)
    _expect_fail(rc.check_rows("u", m["u"].to(dtype), ref["u"], base["u"], dtype)[0], "u", "wrong type row")
