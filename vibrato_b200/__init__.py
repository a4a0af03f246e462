"""vibrato_b200 — H100-native batched Viterbi tokenizer (drop-in for vibrato's tokenisation path).

The package holds only what that path needs: `csrc/` (CUDA kernels + C ABI, built into
libvibrato_b200.so), `api` (host-side mirror of the reference's Rust API over that ABI) and
`synth` (seeded synthetic dictionaries / corpora for tests and benchmarks).
"""
from .api import (BatchResult, Dictionary, SystemDictionaryBuilder, Token, Tokenizer, VibratoError, WordIdx,  # noqa: F401
                  Worker, TOKEN_DTYPE, COMPACT_TOKEN_DTYPE, LEX_TYPE_NAMES, expand_compact_tokens,
                  generate_bigram_info, LatticeNode, LINK_DTYPE, NODE_BEST, SPAN_ANY)

__version__ = "0.1.0"
