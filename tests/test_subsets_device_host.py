"""Host logic of ``subsets=`` on ``VectorBase.search_device`` / ``search_range_device`` on CPU: argument checks
(dtypes, devices, contiguity, the offsets' length, the combinations the device forms refuse), the flags and sizes
passed to ``tav_search_subsets_into`` / ``tav_range_search_subsets_into``, the deferred bookkeeping and a refused
deferred search raising from ``finish_search``.  Tensors are CPU stand-ins that report themselves as CUDA tensors, and
the library is a stand-in that writes the host form's result through their addresses, so no device is needed."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from tests.fake_lib import _view
from tests.test_range_device_host import DevTensor
from tests.test_subsets_host import SUBSETS, SubsetsLib, setup as make_base
from typeagent_py_b200 import _capi


class IntoLib(SubsetsLib):
    """SubsetsLib plus the two device entry points: the host form's result written through the output addresses, or
    a refusal (``refuse``: the status a device check would give) reported now or, deferred, at the finish."""

    def __init__(self, base):
        super().__init__(base)
        self.into_calls = []   # (entry point, n_queries, k or capacity, flags, n_ordinals)
        self.refuse = 0
        self.deferred_error = 0
        self.finishes = 0

    def _status(self, flags):
        if not self.refuse:
            return 0
        if flags & _capi.TAV_DEFER_RETRY:
            self.deferred_error = self.deferred_error or self.refuse
            return 0
        return self.refuse

    def tav_search_subsets_into(self, ix, qp, nq, k, floor, flags, offp, ordp, n_ord, ip, sp, cp, stream):
        self.into_calls.append(("topk", nq, k, flags, n_ord))
        if self.refuse:
            _view(ip, C.c_int64, nq * k)[:] = -1
            _view(sp, C.c_float, nq * k)[:] = 0
            _view(cp, C.c_int32, nq)[:] = 0
            return self._status(flags)
        return self.tav_search_subsets(ix, qp, nq, k, floor, flags & _capi.TAV_TIES_LOW_FIRST, offp, ordp, ip, sp, cp,
                                       stream)

    def tav_range_search_subsets_into(self, ix, qp, nq, floor, flags, offp, ordp, n_ord, cap, op, ip, sp, stream):
        self.into_calls.append(("range", nq, cap, flags, n_ord))
        out = _view(op, C.c_int64, nq + 1)
        if self.refuse:
            out[:] = 0
            return self._status(flags)
        self.tav_range_search_subsets(ix, qp, nq, floor, flags & _capi.TAV_TIES_LOW_FIRST, offp, ordp, op, stream)
        n = min(cap, int(out[-1]))
        if n:
            _view(ip, C.c_int64, n)[:] = self.hits[0][:n]
            _view(sp, C.c_float, n)[:] = self.hits[1][:n]
        return 0

    def tav_finish_search(self, ix, stream, redone):
        self.finishes += 1
        rc, self.deferred_error = self.deferred_error, 0
        return rc

    def tav_last_error(self):
        return b"refused on the device"


@pytest.fixture
def env(monkeypatch):
    base, _, v, q = make_base()
    fake = IntoLib(base)
    base._ensure_device = lambda: (fake, None)
    monkeypatch.setattr(_capi, "load", lambda: fake)  # finish_search and the error text reach the library directly
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: type("S", (), {"cuda_stream": 0})())
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda shape, dtype, device: DevTensor(empty(shape, dtype=dtype), device))
    return base, fake, q


def dev(a, dtype=torch.float32, **kw):
    return DevTensor(torch.from_numpy(np.ascontiguousarray(a)).to(dtype), **kw)


def csr(subsets=SUBSETS, **kw):
    parts = [np.asarray(s, np.int64).reshape(-1) for s in subsets]
    offsets = np.concatenate([[0], np.cumsum([len(p) for p in parts])])
    return dev(offsets, torch.int64, **kw), dev(np.concatenate(parts), torch.int64, **kw)


def test_topk_equals_the_host_form_and_is_not_clamped(env):
    base, fake, q = env
    want_items, want_scores, want_counts = base.search_arrays(q, 200, 0.3, subsets=SUBSETS)
    assert want_items.shape == (5, 134)  # the host form clamps k to the longest subset
    items, scores, counts = base.search_device(dev(q), 200, 0.3, subsets=csr())
    assert items.shape == (5, 200)  # the device form cannot: k stays as asked
    np.testing.assert_array_equal(counts.t.numpy(), want_counts)
    np.testing.assert_array_equal(items.t.numpy()[:, :134], want_items)
    np.testing.assert_array_equal(scores.t.numpy()[:, :134], want_scores)
    assert (items.t.numpy()[:, 134:] == -1).all()
    kind, nq, k, flags, n_ord = fake.into_calls[-1]
    assert (kind, nq, k, n_ord) == ("topk", 5, 200, 189)
    assert flags == _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE and not base._pending


def test_range_equals_the_host_form_under_capacity(env):
    base, fake, q = env
    want = base.search_range(q, 0.3, subsets=SUBSETS, ties_low_first=True)
    total = int(want[0][-1])
    out = (dev(np.zeros(6), torch.int64), dev(np.full(total + 3, -7), torch.int64), dev(np.zeros(total + 3)))
    got = base.search_range_device(dev(q), 0.3, out=out, subsets=csr(), ties_low_first=True)
    assert all(g is o for g, o in zip(got, out))
    np.testing.assert_array_equal(out[0].t.numpy(), want[0])
    np.testing.assert_array_equal(out[1].t.numpy()[:total], want[1])
    assert (out[1].t.numpy()[total:] == -7).all()
    kind, nq, cap, flags, n_ord = fake.into_calls[-1]
    assert (kind, nq, cap, n_ord) == ("range", 5, total + 3, 189)
    assert flags == _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_TIES_LOW_FIRST


def test_flags_passed_through(env):
    base, fake, q = env
    base.force_path = "scan"  # the path options are not flags of the subsets entry points
    base.search_device(dev(q), 4, subsets=csr(), defer_check=True)
    assert fake.into_calls[-1][3] == (_capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_OUTPUTS_ON_DEVICE
                                      | _capi.TAV_DEFER_RETRY)
    base.search_range_device(dev(q), 0.5, 10, subsets=csr(), expected_hits=3)
    assert fake.into_calls[-1][3] == _capi.TAV_QUERIES_ON_DEVICE
    base.search_range_device(dev(q), 0.5, 0, subsets=csr(), defer_check=True, ties_low_first=True)
    assert fake.into_calls[-1][2:4] == (0, _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_DEFER_RETRY
                                        | _capi.TAV_TIES_LOW_FIRST)
    assert base.finish_search() == 0 and fake.finishes == 1


def test_deferred_tensors_kept_until_finish(env):
    base, fake, q = env
    qd, sub = dev(q), csr()
    items, scores, counts = base.search_device(qd, 3, subsets=sub, defer_check=True)
    offsets, r_items, r_scores = base.search_range_device(qd, 0.5, 8, subsets=sub, defer_check=True)
    assert len(base._pending) == 2
    first, second = base._pending
    assert first[0] is qd and first[1] is items and first[2] is scores and first[3] is counts
    assert first[5][0] is sub[0] and first[5][1] is sub[1]
    assert second[1] is r_items and second[2] is r_scores and second[3] is offsets and second[5][0] is sub[0]
    assert base.finish_search() == 0 and fake.finishes == 1 and base._pending == []


@pytest.mark.parametrize("status, exc", [(_capi.TAV_ERR_INVALID, ValueError), (_capi.TAV_ERR_RANGE, IndexError)])
def test_refusals(env, status, exc):
    base, fake, q = env
    fake.refuse = status
    with pytest.raises(exc, match="refused on the device"):
        base.search_device(dev(q), 4, subsets=csr())
    with pytest.raises(exc):
        base.search_range_device(dev(q), 0.5, 10, subsets=csr())
    assert base._pending == []
    # deferred: the calls return, finish_search raises once everything is completed, and nothing stays pending
    items, _, counts = base.search_device(dev(q), 4, subsets=csr(), defer_check=True)
    offsets, _, _ = base.search_range_device(dev(q), 0.5, 10, subsets=csr(), defer_check=True)
    assert (items.t.numpy() == -1).all() and (counts.t.numpy() == 0).all() and (offsets.t.numpy() == 0).all()
    assert len(base._pending) == 2
    with pytest.raises(exc, match="refused on the device"):
        base.finish_search()
    assert base._pending == [] and fake.finishes == 1
    fake.refuse = 0
    assert base.finish_search() == 0 and fake.finishes == 1  # nothing pending: no library call


def test_argument_errors(env):
    base, fake, q = env
    qd = dev(q)
    offsets, ordinals = csr()
    bad = [
        (offsets,),                                                       # not a pair
        (dev(offsets.t.numpy(), torch.int32), ordinals),                   # offsets not int64
        (offsets, dev(ordinals.t.numpy(), torch.float32)),                 # ordinals not int64
        (dev(offsets.t.numpy(), torch.int64, contiguous=False), ordinals),
        (offsets, dev(ordinals.t.numpy(), torch.int64, contiguous=False)),
        (offsets, dev(ordinals.t.numpy(), torch.int64, device="cuda:1")),  # another device
        (dev(offsets.t.numpy(), torch.int64, device="cpu"), ordinals),     # not on a device
        (torch.from_numpy(offsets.t.numpy()), ordinals),                   # a CPU tensor
        (dev(offsets.t.numpy()[:5], torch.int64), ordinals),               # B entries, not B + 1
        (dev(offsets.t.numpy().reshape(6, 1), torch.int64), ordinals),     # 2-D
    ]
    for sub in bad:
        with pytest.raises(ValueError, match="subsets"):
            base.search_device(qd, 4, subsets=sub)
        with pytest.raises(ValueError, match="subsets"):
            base.search_range_device(qd, 0.5, 10, subsets=sub)
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_device(qd, 4, subsets=csr(), allowed=np.ones(400, bool))
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_device(qd, 4, subsets=csr(), row_to_group=dev(np.zeros(400), torch.int32))
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_device(qd, 4, subsets=csr(), item_offset=3)
    with pytest.raises(ValueError, match="k must be"):
        base.search_device(qd, 0, subsets=csr())
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range_device(qd, 0.5, 10, subsets=csr(), subset=[1, 2])
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range_device(qd, 0.5, 10, subsets=csr(), allowed=np.ones(400, bool))
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range_device(qd, 0.5, 10, subsets=csr(), item_offset=1)
    with pytest.raises(ValueError, match="float32"):
        base.search_device(dev(q, torch.float64), 4, subsets=csr())
    assert fake.into_calls == [] and base._pending == []


def test_multi_device_refusal_comes_first(env):
    base, fake, q = env
    base._multi = object()  # a VectorBase over several devices
    with pytest.raises(NotImplementedError):
        base.search_device(dev(q), 4, subsets=(None, None))
    with pytest.raises(NotImplementedError):
        base.search_range_device(dev(q), 0.5, 10, subsets=(None, None))
    base._multi = None


def test_binding_signatures():
    restype, argtypes = _capi.SIGNATURES["tav_search_subsets_into"]
    assert restype is C.c_int and len(argtypes) == 13
    assert argtypes[3] is C.c_int and argtypes[4] is C.c_float and argtypes[8] is C.c_int64
    restype, argtypes = _capi.SIGNATURES["tav_range_search_subsets_into"]
    assert restype is C.c_int and len(argtypes) == 13
    assert argtypes[3] is C.c_float and argtypes[7:9] == [C.c_int64, C.c_int64]
