"""Option classes with the reference's defaults and validation (buffalo/algo/options.py).

The defaults are table-driven here; every value and key matches the cited lines so that option files
written for the reference load unchanged.  ``accelerator`` is accepted for compatibility: this package has
a single, GPU-only backend, so both values select the sm_90a kernels.
"""
from buffalo_b200.misc import aux

_COMMON = dict(evaluation_on_learning=True, compute_loss_on_training=True, early_stopping_rounds=0,
               save_best=False, evaluation_period=1, save_period=10, random_seed=0,
               validation={})                                              # options.py:20-30

_ALS = dict(adaptive_reg=False, save_factors=False, accelerator=False, d=20, num_iters=10, num_workers=1,
            hyper_threads=256, num_cg_max_iters=3, reg_u=0.1, reg_i=0.1, alpha=8.0, optimizer="manual_cg",
            cg_tolerance=1e-10, block_size=32, eps=1e-10, model_path="", data_opt={})   # options.py:66-86

_BPRMF = dict(accelerator=False, use_bias=True, evaluation_period=100, num_workers=1, hyper_threads=256,
              num_iters=100, d=20, update_i=True, update_j=True, reg_u=0.025, reg_i=0.025, reg_j=0.025,
              reg_b=0.025, optimizer="sgd", lr=0.002, min_lr=0.0001, beta1=0.9, beta2=0.999, eps=1e-10,
              per_coordinate_normalize=False, num_negative_samples=1, sampling_power=0.0, verify_neg=True,
              random_positive=False, model_path="", data_opt={})           # options.py:221-252

_WARP = dict(accelerator=False, evaluation_period=5, num_workers=1, hyper_threads=256, num_iters=40, d=64,
             threshold=1.0, score_func="dot", max_trials=500, update_i=True, update_j=True, reg_u=0.0, reg_i=0.0,
             reg_j=0.0, optimizer="adagrad", lr=0.05, min_lr=0.0001, beta1=0.9, beta2=0.999, eps=1e-10,
             per_coordinate_normalize=False, model_path="", data_opt={})   # options.py:286-311

_PLSI = dict(d=20, num_iters=10, num_workers=1, alpha1=1.0, alpha2=1.0, eps=1e-10, model_path="", save_factors=False,
             data_opt={}, inherit_opt={})                                  # options.py:372-384

ALS_OPTIMIZERS = ["llt", "ldlt", "manual_cg", "eigen_cg", "eigen_bicg", "eigen_gmres", "eigen_dgmres",
                  "eigen_minres", "ialspp"]                                 # options.py:90-94
B200_ALS_OPTIMIZERS = ["llt", "ldlt", "manual_cg", "ialspp"]


class AlgoOption(aux.InputOptions):
    _specific = {}

    def get_default_option(self):
        opt = dict(_COMMON)
        opt["validation"] = {}
        opt.update({k: (dict(v) if isinstance(v, dict) else v) for k, v in self._specific.items()})
        return aux.Option(opt) if self._specific else opt

    def is_valid_option(self, opt):
        ok = super().is_valid_option(opt)
        if "num_workers" not in opt:
            raise RuntimeError("num_workers not defined")
        return ok


class ALSOption(AlgoOption):
    _specific = _ALS

    def is_valid_option(self, opt):
        ok = super().is_valid_option(opt)
        if opt.optimizer not in ALS_OPTIMIZERS:
            raise RuntimeError(f"optimizer ({opt.optimizer}) should be in {ALS_OPTIMIZERS}")
        return ok


class BPRMFOption(AlgoOption):
    _specific = _BPRMF


class WARPOption(AlgoOption):
    _specific = _WARP


class PLSIOption(AlgoOption):
    _specific = _PLSI


def _out_of_scope(name):
    class _Opt(AlgoOption):
        def get_default_option(self):
            raise NotImplementedError(name + " is outside the H100 hot-path scope (ALS, BPRMF, WARP, PLSI only)")
    _Opt.__name__ = name
    return _Opt


EALSOption = _out_of_scope("EALSOption")
CFROption = _out_of_scope("CFROption")
W2VOption = _out_of_scope("W2VOption")
