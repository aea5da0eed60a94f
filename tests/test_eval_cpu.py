"""Routing between the host and the device validation paths, and the host-side row gather of the device path."""
import numpy as np
import pytest

from buffalo_b200 import backend
from buffalo_b200.algo.base import Algo
from buffalo_b200.algo.options import ALSOption
from buffalo_b200.evaluate import Evaluable, device
from buffalo_b200.misc import aux


class _Model(Algo, Evaluable):
    """An Evaluable with or without the device hook; the metric paths record that they ran."""

    def __init__(self, hook=True, l2=False):
        Algo.__init__(self)
        self.opt = ALSOption().get_default_option()
        self.opt.validation = aux.Option({"topk": 10})
        self.calls = []
        if hook:
            self._device_eval_model = lambda: device.EvalModel(np.zeros((3, 4), np.float32), np.zeros((5, 4), np.float32),
                                                               None, None, l2)

        class _D(object):
            def has_group(self, name):
                return True
        self.data = _D()

    def normalize(self, group="item"):
        pass

    def _get_feature(self, index, group="item"):
        return None

    def _evaluate_ranking_metrics(self):
        self.calls.append("host-ranking")
        return {"ndcg": 0.0, "map": 0.0, "accuracy": 0.0, "auc": 0.0}

    def _evaluate_score_metrics(self):
        self.calls.append("host-scores")
        return {"rmse": 0.0, "error": 0.0}


@pytest.fixture
def fake_device(monkeypatch):
    calls = []

    class _Evaluation(object):
        def __init__(self, data, model, max_users=None):
            calls.append(("init", max_users))

        def ranking(self, topk, eval_samples):
            calls.append(("ranking", topk))
            return {"ndcg": 1.0, "map": 1.0, "accuracy": 1.0, "auc": 1.0}

        def scores(self):
            calls.append(("scores",))
            return {"rmse": 1.0, "error": 1.0}
    monkeypatch.setattr(backend, "device_available", lambda: True)
    monkeypatch.setattr(device, "Evaluation", _Evaluation)
    return calls


def test_host_path_without_device(monkeypatch):
    monkeypatch.setattr(backend, "device_available", lambda: False)
    m = _Model()
    assert m._device_eval_route() is None
    assert set(m.get_validation_results()) == {"ndcg", "map", "accuracy", "auc", "rmse", "error"}
    assert m.calls == ["host-ranking", "host-scores"]


def test_device_path_routing(fake_device):
    m = _Model()
    m.opt._b200_eval_batch = 64
    assert m.get_validation_results()["ndcg"] == 1.0
    assert m.calls == [] and fake_device == [("init", 64), ("ranking", 10), ("scores",)]


@pytest.mark.parametrize("change", ["option_off", "no_hook", "topk_0", "topk_4097", "topk_missing"])
def test_host_path_when_device_path_declines(fake_device, change):
    m = _Model(hook=change != "no_hook")
    if change == "option_off":
        m.opt._b200_device_eval = False
    elif change.startswith("topk_") and change != "topk_missing":
        m.opt.validation.topk = int(change.split("_")[1])
    elif change == "topk_missing":
        m.opt.validation = aux.Option({"batch": 5})
    assert m._device_eval_route() is None
    m.get_validation_results()
    assert m.calls == ["host-ranking", "host-scores"] and fake_device == []


def test_l2_scores_rank_on_host(fake_device):
    m = _Model(l2=True)
    res = m.get_validation_results()
    assert m.calls == ["host-ranking"] and fake_device == [("init", None), ("scores",)]
    assert res["ndcg"] == 0.0 and res["rmse"] == 1.0
    assert list(res) == ["ndcg", "map", "accuracy", "auc", "rmse", "error"]


def test_trainers_provide_the_hook():
    from buffalo_b200 import ALS, BPRMF, PLSI, WARP
    for cls in (ALS, BPRMF, PLSI, WARP):
        assert callable(getattr(cls, "_device_eval_model", None)), cls


def test_gather_rows_matches_slices():
    rng = np.random.default_rng(0)
    lens = rng.integers(0, 9, size=50)
    lens[[0, 7, 49]] = 0
    indptr = np.cumsum(lens).astype(np.int64)
    keys = rng.integers(0, 1000, size=int(indptr[-1])).astype(np.int32)
    for rows in ([0], [49], [3, 0, 7, 10], rng.choice(50, 20, replace=False), np.arange(50)):
        ptr, got = device._gather_rows(indptr, keys, rows)
        want = [keys[(indptr[r - 1] if r else 0):indptr[r]] for r in rows]
        assert np.array_equal(ptr, np.cumsum([len(w) for w in want]))
        assert np.array_equal(got, np.concatenate(want))
        assert got.dtype == np.int32
