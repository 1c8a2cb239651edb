"""uniter_b200 — H100-native (sm_90a) encoder hot path of ChenRocks/UNITER behind the
reference's own `UniterModel` contract.  See INTEGRATION.md."""
from .model import (UniterConfig, UniterModel, UniterPreTrainedModel,  # noqa: F401
                    register_lengths)
