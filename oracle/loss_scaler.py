"""Host restatement of apex amp's dynamic loss scaler (``LossScaler.update_scale``, dynamic mode), the
policy of every reference driver (train_vqa.py:152,189-199; one scaler per task in pretrain.py:230-233,
298-301), in float32 so that it can be compared bit for bit with ``ub200_adam_prep_scaled``.

    overflow:  scale = max(scale / 2, min_scale) (scale / 2 without a floor), unskipped = 0
    otherwise: unskipped += 1; when unskipped == window: scale = min(scale * 2, max_scale), unskipped = 0

An overflow is what the optimizer's device check sees: the sum of squares of the scaled gradients is
NaN or larger than 3e38 (inf, or about to become inf) — the same test as ``ub200_adam_prep``.
"""
import numpy as np

F32 = np.float32
SUMSQ_LIMIT = F32(3.0e38)


def overflowed(sumsq):
    s = F32(sumsq)
    return bool(np.isnan(s) or abs(s) > SUMSQ_LIMIT)


class LossScaler(object):
    def __init__(self, init_scale=2.**16, scale_window=2000, max_scale=2.**24, min_scale=None):
        self.scale = F32(init_scale)
        self.unskipped = 0
        self.inv_scale = F32(1.0) / self.scale
        self.window = int(scale_window)
        self.max_scale = F32(max_scale)
        self.min_scale = F32(min_scale) if min_scale else None

    def update(self, overflow):
        """One optimizer step whose gradients carry the current scale.  Returns the unscale factor
        of that step (1 / scale before the update)."""
        self.inv_scale = F32(1.0) / self.scale
        if overflow:
            halved = self.scale * F32(0.5)
            self.scale = max(halved, self.min_scale) if self.min_scale is not None else halved
            self.unskipped = 0
        else:
            self.unskipped += 1
            if self.unskipped == self.window:
                self.scale = min(self.scale * F32(2.0), self.max_scale)
                self.unskipped = 0
        return self.inv_scale


class ScaledStepState(object):
    """The device state one fp16 step updates: the optimizer's counters (``ub200_adam_state``: step,
    found_inf, skipped) and the scaler table, one LossScaler per loss id."""

    def __init__(self, scalers):
        self.scalers = list(scalers)
        self.step = 0
        self.skipped = 0
        self.found_inf = 0

    def prep(self, sumsq, loss_id):
        ovf = overflowed(sumsq)
        self.found_inf = int(ovf)
        if ovf:
            self.skipped += 1
        else:
            self.step += 1
        return self.scalers[loss_id].update(ovf)
