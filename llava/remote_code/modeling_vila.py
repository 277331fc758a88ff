"""llava/remote_code/modeling_vila.py:506 — VILAForCausalLM on the sm_90a ops."""
from vila_b200.model.modeling_vila import VILAForCausalLM  # noqa: F401
