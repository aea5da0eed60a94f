"""Deterministic BPRMF / WARP without a GPU: the option key's validation, which comes before the device check, and the
ABI additions."""
import pytest


def _opt(**kw):
    opt = dict(d=16, optimizer="adagrad", deterministic=True)
    opt.update(kw)
    return opt


def test_plain_sgd_is_refused():
    from buffalo_b200 import backend
    g = backend.CuSGD("bpr")
    assert g.init(_opt(optimizer="sgd")) is False
    assert "deterministic" in g.last_error and "Hogwild" in g.last_error and "adagrad" in g.last_error


@pytest.mark.parametrize("kind,optimizer", [("warp", "adagrad"), ("warp", "adam"), ("bpr", "adagrad"),
                                            ("bpr", "adam")])
def test_accumulating_optimizers_accept_the_key(kind, optimizer):
    """Accepted: the option check passes, so init() either succeeds or stops at the device check."""
    import torch
    from buffalo_b200 import _cabi, backend
    g = backend.CuSGD(kind)
    if torch.cuda.is_available():
        assert g.init(_opt(optimizer=optimizer)) is True
        return
    with pytest.raises(_cabi.BackendError) as e:
        g.init(_opt(optimizer=optimizer))
    assert "no CPU fallback" in str(e.value)


def test_key_absent_or_false_keeps_plain_sgd():
    import torch
    from buffalo_b200 import _cabi, backend
    for opt in (dict(d=16, optimizer="sgd"), dict(d=16, optimizer="sgd", deterministic=False)):
        g = backend.CuSGD("bpr")
        if torch.cuda.is_available():
            assert g.init(opt) is True
        else:
            with pytest.raises(_cabi.BackendError):
                g.init(opt)


def test_option_defaults_do_not_list_the_key():
    import buffalo
    for name in ("BPRMFOption", "WARPOption"):
        assert "deterministic" not in getattr(buffalo, name)().get_default_option(), name


def test_segment_length():
    from buffalo_b200 import backend
    assert backend.CuSGD.segment_len() == 4096
