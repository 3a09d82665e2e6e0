"""Host logic of ``VectorBase.search_range_device`` on CPU: argument checks (shapes, dtypes, devices, capacity,
combinations the search refuses), the flags and sizes passed to ``tav_range_search_into``, and the deferred
bookkeeping ``finish_search`` completes.  Tensors are CPU stand-ins that report themselves as CUDA tensors, and
the library is a FakeLib that writes the oracle's hits through their addresses, so no device is needed."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import vectorbase_oracle as O
from tests.fake_lib import _view
from tests.test_range_host import RangeFakeLib, make
from typeagent_py_b200 import _capi


class DevTensor:
    """A contiguous CPU tensor that answers like a CUDA tensor on `device` (the library only sees addresses)."""

    def __init__(self, t: torch.Tensor, device="cuda:0", contiguous=True):
        self.t, self.device, self._contiguous = t, torch.device(device), contiguous
        self.is_cuda = self.device.type == "cuda"
        self.dtype, self.shape = t.dtype, t.shape

    def is_contiguous(self):
        return self._contiguous

    def dim(self):
        return self.t.dim()

    def numel(self):
        return self.t.numel()

    def data_ptr(self):
        return self.t.data_ptr()


class IntoFakeLib(RangeFakeLib):
    """RangeFakeLib plus tav_range_search_into (its hits through the output addresses, first `cap` of them)."""

    def __init__(self, base):
        super().__init__(base)
        self.into_calls = []    # (n_queries, flags, subset_len, item_offset, expected_hits, capacity)
        self.finishes = 0

    def tav_range_search_into(self, ix, qp, nq, floor, flags, sub_ptr, sub_len, item_offset, expected, cap, op, ip, sp,
                              stream):
        self.into_calls.append((nq, flags, sub_len, item_offset, expected, cap))
        offsets = np.zeros(nq + 1, np.int64)
        self.tav_range_search(ix, qp, nq, floor, flags, sub_ptr, sub_len, item_offset, expected,
                              offsets.ctypes.data_as(C.c_void_p), stream)
        _view(op, C.c_int64, nq + 1)[:] = offsets
        n = min(cap, int(offsets[-1]))
        if n:
            _view(ip, C.c_int64, n)[:] = np.asarray(self.hits[0][:n], np.int64) + item_offset
            _view(sp, C.c_float, n)[:] = self.hits[1][:n]
        return 0

    def tav_set_query_masks(self, ix, words, n_queries, n_rows, words_per, on_device, stream):
        return 0

    def tav_finish_search(self, ix, stream, redone):
        self.finishes += 1
        return 0


@pytest.fixture
def setup(monkeypatch):
    v, q = O.make_corpus(300, 16, seed=21, n_queries=3)
    base, _ = make(v)
    fake = IntoFakeLib(base)
    base._ensure_device = lambda: (fake, None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: type("S", (), {"cuda_stream": 0})())
    empty = torch.empty
    monkeypatch.setattr(torch, "empty", lambda shape, dtype, device: DevTensor(empty(shape, dtype=dtype), device))
    return base, fake, v, q


def dev(a, dtype=torch.float32, **kw):
    return DevTensor(torch.from_numpy(np.ascontiguousarray(a)).to(dtype), **kw)


def outs(b, cap, **kw):
    return (dev(np.zeros(b + 1), torch.int64, **kw), dev(np.full(cap, -7), torch.int64),
            dev(np.zeros(cap), torch.float32))


def test_result_through_the_library(setup):
    base, fake, v, q = setup
    want = base.search_range(q, 0.55)
    total = int(want[0][-1])
    out = outs(3, total + 5)
    got = base.search_range_device(dev(q), 0.55, out=out)
    assert all(g is o for g, o in zip(got, out))
    np.testing.assert_array_equal(out[0].t.numpy(), want[0])
    np.testing.assert_array_equal(out[1].t.numpy()[:total], want[1])
    assert (out[1].t.numpy()[total:] == -7).all()
    nq, flags, sub_len, item_offset, expected, cap = fake.into_calls[-1]
    assert (nq, sub_len, item_offset, cap) == (3, 0, 0, total + 5)
    assert expected == cap  # expected_hits defaults to the capacity
    assert flags == _capi.TAV_QUERIES_ON_DEVICE and not base._pending


def test_flags_and_sizes_passed_through(setup):
    base, fake, v, q = setup
    base.force_path = "scan2"  # the two-kernel top-k scan has no threshold form: FORCE_SCAN only
    base.search_range_device(dev(q), 0.5, 10, ties_low_first=True, expected_hits=77, item_offset=5)
    nq, flags, _, item_offset, expected, cap = fake.into_calls[-1]
    assert flags == _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_FORCE_SCAN | _capi.TAV_TIES_LOW_FIRST
    assert (item_offset, expected, cap) == (5, 77, 10)
    base.force_path = "mma"
    base.search_range_device(dev(q), 0.5, 10, allowed=np.arange(300) % 2 == 0)
    assert fake.into_calls[-1][1] == _capi.TAV_QUERIES_ON_DEVICE | _capi.TAV_FORCE_MMA | _capi.TAV_USE_ROW_MASK
    base.search_range_device(dev(q), 0.5, 10, allowed=np.ones((3, 300), bool))
    assert fake.into_calls[-1][1] & _capi.TAV_USE_QUERY_MASKS
    base.search_range_device(dev(q), 0.5, 10, subset=[4, 2, 2])
    assert fake.into_calls[-1][2] == 3


def test_deferred_tensors_kept_until_finish(setup, monkeypatch):
    base, fake, v, q = setup
    monkeypatch.setattr(_capi, "load", lambda: fake)  # finish_search reaches the library directly
    qd = dev(q)
    got = base.search_range_device(qd, 0.5, 20, defer_check=True)
    assert fake.into_calls[-1][1] & _capi.TAV_DEFER_RETRY
    assert len(base._pending) == 1 and base._pending[0][0] is qd and base._pending[0][1] is got[1]
    base.search_range_device(qd, 0.5, 20, defer_check=True)
    assert base.finish_search() == 0 and fake.finishes == 1 and base._pending == []


def test_argument_errors(setup):
    base, fake, v, q = setup
    bad_queries = [
        torch.from_numpy(q),                            # a CPU tensor
        dev(q, torch.float64),                          # not float32
        dev(q, contiguous=False),
        dev(q[:, :8]),                                  # wrong width
        dev(q[0]),                                      # 1-D
        q,                                              # numpy
    ]
    for bad in bad_queries:
        with pytest.raises(ValueError):
            base.search_range_device(bad, 0.5, 10)
    qd = dev(q)
    for cap in (-1, 2.5, True):
        with pytest.raises(ValueError, match="capacity"):
            base.search_range_device(qd, 0.5, cap)
    with pytest.raises(ValueError, match="capacity is needed"):
        base.search_range_device(qd, 0.5)
    with pytest.raises(ValueError, match="expected_hits"):
        base.search_range_device(qd, 0.5, 10, expected_hits=-1)
    bad_outs = [
        outs(2, 10),                                                            # offsets of the wrong length
        (dev(np.zeros(4), torch.int32),) + outs(3, 10)[1:],                     # offsets not int64
        outs(3, 10)[:1] + (dev(np.zeros(10), torch.float32),) + outs(3, 10)[2:],  # items not int64
        outs(3, 10)[:2] + (dev(np.zeros(10), torch.float64),),                  # scores not float32
        outs(3, 10)[:2],                                                        # two tensors
        (dev(np.zeros(4), torch.int64, device="cuda:1"),) + outs(3, 10)[1:],    # another device
        (dev(np.zeros(4), torch.int64, device="cpu"),) + outs(3, 10)[1:],       # not on the device
        outs(3, 4),                                                             # room for 4 < capacity
    ]
    for out in bad_outs:
        with pytest.raises(ValueError):
            base.search_range_device(qd, 0.5, 10, out=out)
    with pytest.raises(ValueError, match="cannot be combined"):
        base.search_range_device(qd, 0.5, 10, subset=[1, 2], allowed=np.ones(300, bool))
    with pytest.raises(IndexError):
        base.search_range_device(qd, 0.5, 10, subset=[1.5])
    with pytest.raises(ValueError):
        base.search_range_device(qd, 0.5, 10, allowed=np.ones(299, bool))   # mask of the wrong length
    with pytest.raises(ValueError):
        base.search_range_device(qd, 0.5, 10, allowed=np.ones((2, 300), bool))  # masks for 2 of 3 queries
    assert fake.into_calls == [] and base._pending == []


def test_capacity_defaults_to_the_room_in_out(setup):
    base, fake, v, q = setup
    base.search_range_device(dev(q), 0.5, out=outs(3, 12))
    assert fake.into_calls[-1][5] == 12
    base.search_range_device(dev(q), 0.5, 5, out=outs(3, 12))
    assert fake.into_calls[-1][5] == 5


def test_binding_signature():
    restype, argtypes = _capi.SIGNATURES["tav_range_search_into"]
    assert restype is C.c_int and len(argtypes) == 14
    assert argtypes[3] is C.c_float and argtypes[7:10] == [C.c_int64, C.c_int64, C.c_int64]
