from buffalo_b200.parallel.base import (ParALS, ParBPRMF, ParCFR, ParW2V, cap_categories, dot_topn, quickselect,
                                        rerank_mmr)
