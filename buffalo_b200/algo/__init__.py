# superset of the reference's (empty) buffalo/algo/__init__.py so that examples/example_als.py's
# `from buffalo.algo import ALS, ALSOption` works (SURVEY.md 0-10)
from buffalo_b200.algo.als import ALS, inited_CUALS
from buffalo_b200.algo.base import Algo, Serializable
from buffalo_b200.algo.bpr import BPRMF, inited_CUBPR
from buffalo_b200.algo.options import AlgoOption, ALSOption, BPRMFOption, PLSIOption, WARPOption
from buffalo_b200.algo.plsi import PLSI
from buffalo_b200.algo.warp import WARP
