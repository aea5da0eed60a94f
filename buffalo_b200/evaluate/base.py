"""Ranking / score metrics on the held-out split (buffalo/evaluate/base.py:44-148): NDCG, MAP,
accuracy (= |topk & gt| / |gt|, :93), AUC, RMSE/error.  Top-k selection uses argpartition instead of the
reference's OpenMP quickselect (buffalo/parallel/_core.hpp:69-86) -- per-evaluation work on <= 500 rows."""
import numpy as np


def topk_indices(scores, k, ordered=True):
    """indices of the k largest entries per row, best first."""
    scores = np.asarray(scores)
    k = min(k, scores.shape[1])
    part = np.argpartition(-scores, k - 1, axis=1)[:, :k]
    if ordered:
        vals = np.take_along_axis(scores, part, axis=1)
        part = np.take_along_axis(part, np.argsort(-vals, axis=1, kind="stable"), axis=1)
    return part.astype(np.int32)


class Evaluable(object):
    def __init__(self, *args, **kwargs):
        pass

    def prepare_evaluation(self):
        if not self.opt.validation or not self.data.has_group("vali"):
            return
        if not hasattr(self.data, "vali_data"):
            self.data._prepare_validation_data()

    def show_validation_results(self):
        res = self.get_validation_results()
        if not res:
            return "No validation results"
        return "Validation results: " + ", ".join(f"{k}: {v:0.5f}" for k, v in res.items())

    def get_validation_results(self):
        if not self.opt.validation or not self.data.has_group("vali"):
            return
        model = self._device_eval_route()
        res = {}
        if model is None:
            res.update(self._evaluate_ranking_metrics())
            res.update(self._evaluate_score_metrics())
            return res
        from buffalo_b200.evaluate.device import Evaluation
        if model.l2:   # ranking by 1 - |p - q|^2 has no device top-k: host ranking, device score metrics
            res.update(self._evaluate_ranking_metrics())
        ev = Evaluation(self.data, model, max_users=self.opt.get("_b200_eval_batch"))
        if not model.l2:
            res.update(ev.ranking(self.opt.validation.topk, self.opt.validation.eval_samples))
        res.update(ev.scores())
        return res

    def evaluate(self, test, cutoffs=(10,), exclude_seen=True, diversity=False, per_user=False):
        """Ranking metrics of this model on held-out interactions, on the GPU (DESIGN.md 4.14).

        test: a scipy sparse (num_users, num_items) matrix in the model's index space; row u's ground truth is its
        distinct columns with a nonzero value after duplicates are summed, and only users with at least one are
        evaluated.  Each is ranked once at the largest cutoff by the masked top-k of the validation path, leaving out
        exclude_seen's items as ParALS.topk_recommendation does: True the rows of the attached training data, False
        nothing, a scipy sparse (num_users, num_items) matrix its rows.  cutoffs: integers in [1, 4096] (<= 256 with
        diversity).  diversity=True adds ild@K over the rows of the item factors Q.  The result is evaluate_lists'
        for those lists.  Unlike get_validation_results(), users without training items are evaluated too.  Not for
        WARP with score_func="l2", which has no device ranking.  GPU only: without one the
        backend's "no CPU fallback" error is raised after the argument checks."""
        from buffalo_b200.evaluate.offline import evaluate_model
        return evaluate_model(self, test, cutoffs, exclude_seen, diversity, per_user)

    def _device_eval_route(self):
        """The EvalModel of the device path (evaluate/device.py), or None for the host path: the device path needs a
        trainer that provides _device_eval_model, 0 < topk <= 4096, a GPU, and the private option _b200_device_eval
        not False."""
        hook = getattr(self, "_device_eval_model", None)
        topk = self.opt.validation.get("topk")
        if hook is None or self.opt.get("_b200_device_eval") is False or not isinstance(topk, (int, np.integer)) \
                or not 0 < topk <= 4096:
            return None
        from buffalo_b200 import backend
        if not backend.device_available():
            return None
        return hook()

    def get_topk(self, scores, k, sorted=True, num_threads=4):
        scores = np.asarray(scores)
        single = scores.ndim == 1
        if single:
            scores = scores.reshape(1, -1)
        assert min(k, scores.shape[1]) > 0, f"k({k}) or cols({scores.shape[1]}) should be greater than 0"
        out = topk_indices(scores, k, ordered=sorted)
        return out[0] if single else out

    def _evaluate_ranking_metrics(self):
        if not hasattr(self.data, "vali_data"):
            self.prepare_evaluation()
        v = self.data.vali_data
        batch = self.opt.validation.get("batch", 128)
        topk = self.opt.validation.topk
        gt, rows, seen_of = v["vali_gt"], v["vali_rows"], v["validation_seen"]
        num_items = self.data.get_header()["num_items"]
        if self.opt.validation.eval_samples:
            rows = np.random.choice(rows, size=min(self.opt.validation.eval_samples, len(rows)), replace=False)
        gains = 1.0 / np.log2(np.arange(2, topk + 2))
        ideal = np.cumsum(gains)
        tot = dict(ndcg=0.0, map=0.0, accuracy=0.0, auc=0.0)
        count = 0.0
        for s in range(0, len(rows), batch):
            recs = self._get_topk_recommendation(rows[s:s + batch], topk=topk + v["validation_max_seen_size"])
            for row, cand in recs:
                seen = seen_of.get(row, set())
                if not seen:
                    continue
                ranked = [c for c in cand if c not in seen][:topk]
                truth = gt[row]
                hits = np.array([1.0 if r in truth else 0.0 for r in ranked])
                tot["accuracy"] += len(set(ranked) & truth) / len(truth)
                cum_hits = np.cumsum(hits)
                dcg = float((hits * gains[:len(hits)]).sum())
                ap = float((hits * cum_hits / np.arange(1, len(hits) + 1)).sum())
                n_pos, miss = len(truth), float((1 - hits).sum())
                n_neg = num_items - n_pos
                auc = float(((1 - hits) * cum_hits).sum()) + ((cum_hits[-1] if len(hits) else 0.0) + n_pos) / 2.0 * (n_neg - miss)
                tot["auc"] += auc / (n_pos * n_neg)
                tot["ndcg"] += dcg / ideal[min(n_pos, topk) - 1]
                tot["map"] += ap / min(n_pos, topk)
                count += 1.0
        return {k: val / count for k, val in tot.items()}

    def _evaluate_score_metrics(self):
        if not hasattr(self.data, "vali_data"):
            self.prepare_evaluation()
        v = self.data.vali_data
        err = np.asarray(self._get_scores(v["row"], v["col"]), dtype=np.float64) - v["val"]
        return {"rmse": float(np.sqrt(np.mean(err ** 2))), "error": float(np.mean(np.abs(err)))}
