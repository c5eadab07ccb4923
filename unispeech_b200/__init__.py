"""unispeech_b200 -- WavLM / UniSpeech-SAT encoder hot path for the H100 (hand-written sm_90a kernels behind a C ABI)."""

__version__ = "0.1.0"
