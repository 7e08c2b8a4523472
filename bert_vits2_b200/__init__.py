"""bert_vits2_b200 — Hopper-native (sm_90a) VITS2 inference engine behind the Bert-VITS2 `SynthesizerTrn.infer` API."""
from .spec import ModelConfig, param_specs, param_shapes  # noqa: F401

__all__ = ["ModelConfig", "param_specs", "param_shapes"]
