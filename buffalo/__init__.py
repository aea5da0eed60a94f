"""`buffalo` -- import alias of buffalo_b200, so that code written for kakao/buffalo
(examples/example_als.py, benchmark/test_performance.py) runs unchanged on the H100 backend.
Every submodule path of the reference that the hot path's callers use is mapped onto buffalo_b200."""
import importlib
import sys

import buffalo_b200
from buffalo_b200 import *  # noqa: F401,F403
from buffalo_b200 import __version__  # noqa: F401

_ALIASES = {
    "buffalo.algo": "buffalo_b200.algo", "buffalo.algo.als": "buffalo_b200.algo.als",
    "buffalo.algo.bpr": "buffalo_b200.algo.bpr", "buffalo.algo.warp": "buffalo_b200.algo.warp",
    "buffalo.algo.plsi": "buffalo_b200.algo.plsi",
    "buffalo.algo.base": "buffalo_b200.algo.base", "buffalo.algo.options": "buffalo_b200.algo.options",
    "buffalo.data": "buffalo_b200.data", "buffalo.data.base": "buffalo_b200.data.base",
    "buffalo.data.mm": "buffalo_b200.data.mm", "buffalo.data.stream": "buffalo_b200.data.stream",
    "buffalo.data.prepro": "buffalo_b200.data.prepro", "buffalo.data.buffered_data": "buffalo_b200.data.buffered_data",
    "buffalo.evaluate": "buffalo_b200.evaluate", "buffalo.evaluate.base": "buffalo_b200.evaluate.base",
    "buffalo.misc": "buffalo_b200.misc", "buffalo.misc.aux": "buffalo_b200.misc.aux",
    "buffalo.misc._aux": "buffalo_b200.misc.aux", "buffalo.misc.util": "buffalo_b200.misc.aux",
    "buffalo.misc.log": "buffalo_b200.misc.log",
    "buffalo.parallel": "buffalo_b200.parallel", "buffalo.parallel.base": "buffalo_b200.parallel.base",
}
for _alias, _target in _ALIASES.items():
    sys.modules[_alias] = importlib.import_module(_target)
algo, data, evaluate, misc, parallel = (sys.modules["buffalo." + n] for n in ("algo", "data", "evaluate", "misc", "parallel"))
