"""metrabs_b200: H100 (sm_90a) implementation of the MeTRAbs per-crop inference hot path behind the
metrabs_pytorch ``Metrabs.forward`` API.  Compute lives in libmetrabs_b200.so (hand-written CUDA behind a C ABI,
include/metrabs_b200.h); this package is the host-side mirror of the reference interface."""
from metrabs_b200.util import Config, get_config, set_config  # noqa: F401
from metrabs_b200._lib import MetrabsB200Error, lib  # noqa: F401
