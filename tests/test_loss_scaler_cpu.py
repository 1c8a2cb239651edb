"""CPU: the host restatement of apex's dynamic loss-scaling policy (oracle/loss_scaler.py) on
hand-worked sequences, and the host side of uniter_b200.optim.DynamicLossScaler (table layout,
apex-compatible state_dict)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle.loss_scaler import LossScaler, ScaledStepState, overflowed

INF, NAN = float("inf"), float("nan")


def test_apex_defaults():
    s = LossScaler()
    assert s.scale == 2.**16 and s.window == 2000 and s.max_scale == 2.**24 and s.min_scale is None


def test_overflow_halves_the_scale_and_resets_the_counter():
    s = LossScaler(init_scale=1024.0, scale_window=5)
    for _ in range(3):
        s.update(False)
    assert (s.scale, s.unskipped) == (1024.0, 3)
    inv = s.update(True)
    assert inv == np.float32(1 / 1024.0)          # the overflowed step carried the old scale
    assert (s.scale, s.unskipped) == (512.0, 0)
    # the window starts again from zero: 4 clean steps do not double, the 5th does
    for _ in range(4):
        s.update(False)
    assert (s.scale, s.unskipped) == (512.0, 4)
    assert s.update(False) == np.float32(1 / 512.0)
    assert (s.scale, s.unskipped) == (1024.0, 0)


def test_2000_clean_steps_double_the_scale():
    s = LossScaler()
    for _ in range(1999):
        s.update(False)
    assert (s.scale, s.unskipped) == (2.**16, 1999)
    s.update(False)
    assert (s.scale, s.unskipped) == (2.**17, 0)
    for _ in range(2000):
        s.update(False)
    assert s.scale == 2.**18


def test_the_cap_holds():
    s = LossScaler(init_scale=2.**23, scale_window=2)
    for _ in range(2):
        s.update(False)
    assert s.scale == 2.**24
    for _ in range(10):
        s.update(False)
    assert (s.scale, s.unskipped) == (2.**24, 0)
    s.update(True)
    assert s.scale == 2.**23


def test_the_optional_floor_holds():
    s = LossScaler(init_scale=8.0, scale_window=100, min_scale=2.0)
    scales = []
    for _ in range(5):
        s.update(True)
        scales.append(float(s.scale))
    assert scales == [4.0, 2.0, 2.0, 2.0, 2.0]
    s = LossScaler(init_scale=8.0, scale_window=100)           # no floor: keeps halving
    for _ in range(5):
        s.update(True)
    assert s.scale == 0.25
    assert LossScaler(min_scale=0.0).min_scale is None          # apex: a zero floor is no floor


def test_nan_and_inf_count_as_overflow():
    assert overflowed(INF) and overflowed(-INF) and overflowed(NAN)
    assert overflowed(3.1e38)                       # the device check's limit (ub200_adam_prep)
    assert not overflowed(0.0) and not overflowed(2.9e38) and not overflowed(1e-30)
    st = ScaledStepState([LossScaler(init_scale=64.0, scale_window=3)])
    st.prep(1.0, 0)
    st.prep(NAN, 0)
    assert (st.step, st.skipped, st.found_inf) == (1, 1, 1)
    assert (st.scalers[0].scale, st.scalers[0].unskipped) == (32.0, 0)
    st.prep(2.0, 0)
    assert (st.step, st.skipped, st.found_inf) == (2, 1, 0)


def test_only_the_stepped_loss_id_moves():
    st = ScaledStepState([LossScaler(init_scale=2.**10, scale_window=2), LossScaler(init_scale=2.**30)])
    st.prep(1.0, 0)
    st.prep(INF, 1)
    assert (st.scalers[0].scale, st.scalers[0].unskipped) == (2.**10, 1)
    assert (st.scalers[1].scale, st.scalers[1].unskipped) == (2.**29, 0)
    st.prep(1.0, 0)
    assert (st.scalers[0].scale, st.scalers[0].unskipped) == (2.**11, 0)
    assert st.scalers[1].scale == 2.**29


def test_device_table_layout_and_state_dict_on_the_host():
    from uniter_b200 import _lib
    from uniter_b200.optim import DynamicLossScaler
    assert C.sizeof(_lib.LossScalerEntry) == 32          # == sizeof(ub200_loss_scaler)
    sc = DynamicLossScaler(num_losses=3, init_scale=2.**20, scale_window=7, max_scale=2.**22, min_scale=4.0,
                           device="cpu")
    ints = sc.table.view(torch.int32)
    assert sc.table.shape == (3, 8)
    for k in range(3):
        assert sc.table[k, 0] == 2.**20 and ints[k, 1] == 0 and sc.table[k, 2] == 2.**-20
        assert ints[k, 3] == 7 and sc.table[k, 4] == 2.**22 and sc.table[k, 5] == 4.0
    loss = torch.tensor(0.75, dtype=torch.float16)
    assert sc.scale(loss, 1).dtype == torch.float32 and sc.scale(loss, 1).item() == 0.75 * 2.**20
    with pytest.raises(IndexError):
        sc.scale(loss, 3)
    # apex amp.state_dict() layout: 'loss_scaler<k>': {'loss_scale', 'unskipped'}
    sd = {"loss_scaler0": {"loss_scale": 512.0, "unskipped": 3},
          "loss_scaler1": {"loss_scale": 2.**24, "unskipped": 0},
          "loss_scaler2": {"loss_scale": 8.0, "unskipped": 6}}
    addr = sc.table.data_ptr()
    sc.load_state_dict(sd)
    assert sc.table.data_ptr() == addr                    # loaded in place: captured graphs stay valid
    assert sc.state_dict() == sd
    assert sc.loss_scale(2) == 8.0 and sc.unskipped(2) == 6 and ints[2, 3] == 7
    assert sc.table[0, 2] == 1.0 / 512.0
    with pytest.raises(ValueError):
        sc.load_state_dict({"loss_scaler0": sd["loss_scaler0"]})
    assert math.isclose(DynamicLossScaler(device="cpu").loss_scale(), 65536.0)
