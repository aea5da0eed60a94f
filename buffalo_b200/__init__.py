"""buffalo_b200 -- H100-native implementation of kakao/buffalo's matrix-factorisation training hot path
(ALS row solves, BPRMF / WARP negative-sampling SGD, pLSI EM) behind buffalo's own Python API.

The compute lives in buffalo_b200/csrc (hand-written sm_90a CUDA behind the C ABI of
include/buffalo_b200.h).  There is no CPU fallback.  `import buffalo` resolves to this package
(see the `buffalo/` alias at the repository root), so scripts written for the reference run unchanged.
"""
__version__ = "0.1.0"

from buffalo_b200.algo.als import ALS, inited_CUALS
from buffalo_b200.algo.base import Algo
from buffalo_b200.algo.bpr import BPRMF, inited_CUBPR
from buffalo_b200.algo.options import (AlgoOption, ALSOption, BPRMFOption, CFROption, EALSOption, PLSIOption,
                                       W2VOption, WARPOption)
from buffalo_b200.algo.plsi import PLSI
from buffalo_b200.algo.warp import WARP
from buffalo_b200.data.mm import MatrixMarket, MatrixMarketOptions
from buffalo_b200.data.stream import Stream, StreamOptions
from buffalo_b200.misc import aux, log, set_log_level
from buffalo_b200.parallel.base import ParALS, ParBPRMF, ParCFR, ParW2V


def _out_of_scope(name):
    class _Algo(object):
        def __init__(self, *a, **k):
            raise NotImplementedError(name + " is outside the H100 hot-path scope (ALS, BPRMF, WARP, PLSI only)")
    _Algo.__name__ = name
    return _Algo


CFR, EALS, W2V = (_out_of_scope(n) for n in ("CFR", "EALS", "W2V"))
