"""The window kernels (b2_window_heads / positions / scan / rmq / frame / invert, include/b200sql.h) against NumPy:
the positions word for word, and every function through executor._WindowSpecRun against tests/window_ref.py, at
n around the warp and the 2048-row scan tile, one partition over every tile and all one-row partitions, with
+-inf, NaN and -0.0 in keys and values, int64 wrap, and MIN / MAX frames up to w = 10^5."""
import numpy as np
import pytest
import torch

from tests import query_ref as Q
from tests import window_ref as W

pytestmark = pytest.mark.gpu
INF = float("inf")
TILE = 2048
SIZES = [1, 31, 32, 33, TILE - 1, TILE + 1, 5 * TILE + 7]


def _part(cols):
    from dask_sql_b200 import device as D
    from dask_sql_b200.executor import Part
    torch.cuda.set_device(0)
    out = Part({}, len(next(iter(cols.values()))))
    for name, a in cols.items():
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        out[name] = D.DeviceColumn(t, None, D.F64 if a.dtype == np.float64 else D.I64)
    return out


def _host(col):
    data = col.data.cpu().numpy()
    if col.valid is None:
        return data, np.zeros(len(data), bool)
    bits = np.unpackbits(col.valid.cpu().numpy().view(np.uint8), bitorder="little")[:len(data)]
    return data, bits == 0


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("layout", ["one", "singletons", "random"])
def test_positions(n, layout):
    from dask_sql_b200.executor import _WindowSpecRun
    rng = np.random.default_rng(n)
    k = {"one": np.zeros(n, np.int64), "singletons": rng.permutation(n).astype(np.int64),
         "random": rng.integers(0, max(1, n // 7), n)}[layout]
    t = rng.integers(0, 4, n)
    run = _WindowSpecRun(_part({"k": k, "t": t}), ["k"], [("t", True, False)])
    torch.cuda.synchronize()
    idx = run.idx.cpu().numpy()
    perm = np.lexsort((t, k))
    assert np.array_equal(idx, perm)
    ps, qs, dn, pend, qend = (p.cpu().numpy() for p in run.pos)
    ks, ts = k[perm], t[perm]
    phead = np.r_[True, ks[1:] != ks[:-1]]
    qhead = phead | np.r_[True, ts[1:] != ts[:-1]]
    pos = np.arange(n)
    exp_ps = np.maximum.accumulate(np.where(phead, pos, 0))
    exp_qs = np.maximum.accumulate(np.where(qhead, pos, 0))
    assert np.array_equal(ps, exp_ps) and np.array_equal(qs, exp_qs)
    cq = np.cumsum(qhead)
    assert np.array_equal(dn, cq - cq[exp_ps] + 1)
    pend_exp = np.r_[np.flatnonzero(phead)[1:] - 1, n - 1]
    qend_exp = np.r_[np.flatnonzero(qhead)[1:] - 1, n - 1]
    assert np.array_equal(pend[np.flatnonzero(phead)], pend_exp)
    assert np.array_equal(qend[np.flatnonzero(qhead)], qend_exp)


FUNCS = [("ROW_NUMBER", None), ("RANK", None), ("DENSE_RANK", None), ("COUNT", None), ("COUNT", "v"), ("SUM", "x"),
         ("SUM", "f"), ("AVG", "x"), ("MIN", "v"), ("MAX", "v"), ("FIRST_VALUE", "v"), ("LAST_VALUE", "x")]
FRAMES = [(True, -INF, 0), (True, 0, INF), (True, 0, 0), (False, -INF, INF), (False, -3, 2), (False, 0, INF),
          (False, 2, 5), (False, -5, -2), (False, -40, 40), (False, 2, 1), (False, -1, -3)]   # the last two: empty


def _check(rel, cols, partition, order, fn, arg, frame, what):
    from dask_sql_b200.executor import _WindowSpecRun
    from dask_sql_b200.device import gather
    run = _WindowSpecRun(_part(cols), partition, order)
    col = run.function(fn.lower(), arg, frame)
    inv = torch.empty(run.n, dtype=torch.int32, device="cuda")
    from dask_sql_b200 import _lib as L, device as D
    L.window_invert(D.ptr(run.idx), run.n, D.ptr(inv), D.stream_ptr())
    data, null = _host(gather(col, inv, False))
    kind, exp = W.window(rel, partition, order, fn, arg, frame)
    got = [None if nl else (float(x) if kind in ("float", "bounded") else int(x)) for x, nl in zip(data, null)]
    if kind in ("float", "bounded"):
        got = [np.nan if g is None else g for g in got]
    Q.assert_result({"o": got}, Q.Result({"o": exp}, {"o": kind}), what=what)


@pytest.mark.parametrize("n", SIZES)
def test_functions_and_frames(n):
    rng = np.random.default_rng(100 + n)
    k = rng.integers(0, max(1, n // 50), n).astype(np.float64)
    k[rng.random(n) < 0.05] = np.nan
    if n > 3:
        k[:3] = [0.0, -0.0, INF]
    t = rng.integers(0, 9, n)
    v = rng.normal(0, 10, n)
    v[rng.random(n) < 0.1] = np.nan
    if n > 5:
        v[3:6] = [INF, -0.0, 0.0]
    x = rng.integers(-(1 << 62), 1 << 62, n) * 3                 # int64 sums wrap
    f = rng.integers(-999, 999, n) / 16.0
    cols = {"k": k, "t": t, "v": v, "x": x, "f": f, "u": np.arange(n)}
    rel = {name: Q.Column(a, None, Q.F64 if a.dtype == np.float64 else Q.I64) for name, a in cols.items()}
    order = [("t", True, False), ("u", True, False)]
    for fn, arg in FUNCS:
        for frame in (FRAMES if fn not in ("ROW_NUMBER", "RANK", "DENSE_RANK") else [None]):
            o = order if fn not in ("RANK", "DENSE_RANK") else [("t", True, False)]
            _check(rel, cols, ["k"], o, fn, arg, frame or (True, -INF, 0), f"{fn}({arg}) {frame} n={n}")


@pytest.mark.parametrize("w", [1, 2, 17, 1000, 100_000])
def test_minmax_wide_frames(w):
    n = 250_000
    rng = np.random.default_rng(w)
    v = rng.normal(size=n)
    cols = {"k": np.zeros(n, np.int64), "u": np.arange(n), "v": v}
    from dask_sql_b200.executor import _WindowSpecRun
    run = _WindowSpecRun(_part(cols), ["k"], [("u", True, False)])
    for fn in ("min", "max"):
        col = run.function(fn, "v", (False, -(w - 1), 0))
        got, null = _host(col)                                    # one partition in input order: no scatter
        assert not null.any()
        from numpy.lib.stride_tricks import sliding_window_view
        pad = np.r_[np.full(w - 1, np.inf if fn == "min" else -np.inf), v]
        exp = getattr(sliding_window_view(pad, w), fn)(axis=1)
        assert np.array_equal(got, exp), fn


def test_argument_checks():
    """rejected before any launch; the buffers are real allocations all the same, and n = 0 launches nothing"""
    import ctypes
    from dask_sql_b200 import _lib as L
    from dask_sql_b200 import device as D
    torch.cuda.set_device(0)
    f = L.WinFrame()
    f.fn, f.n = 99, 0
    with pytest.raises(L.B200SqlError, match="null argument|bad window function"):
        L.window_frame(ctypes.byref(f), D.stream_ptr())
    n = 4
    flags = torch.zeros(n, dtype=torch.uint8, device="cuda")
    data = torch.zeros(n, dtype=torch.int64, device="cuda")
    out = torch.zeros(n, dtype=torch.int64, device="cuda")
    ws = torch.zeros(L.window_ws_bytes(n), dtype=torch.uint8, device="cuda")
    col = L.Col()
    col.data, col.dtype = D.ptr(data).value, L.I64
    pre = L.WinPrefix()
    pre.val = D.ptr(out).value
    with pytest.raises(L.B200SqlError, match="seg_mask"):
        L.window_scan(D.ptr(flags), ctypes.byref(col), n, L.WIN_SUM_I, 3, 0, ctypes.byref(pre), D.ptr(ws),
                      D.stream_ptr())
