"""aha_b200 -- B200-native (sm_100a) prefill + decode path for Qwen3 / Qwen3-VL / Qwen3-ASR behind
jhqxxx/aha's InferenceModel seam.  The compute lives in libaha_b200.so (hand-written CUDA, C ABI in
include/aha_b200.h); this package is the Python host-side mirror used by tests and bench.py."""
from .inference import B200Error, B200Model, MultiModalData, fsm_check, nccl_unique_id, rope_index, rules_check  # noqa: F401
