"""The image reductions (csrc/reduction.cu, `ImageReducer` / `rmd_reduce_*`) against exact references.

Integers are checked against Python integers; float sums against math.fsum (the exact sum rounded once to double),
itself checked with fractions.Fraction on small cases.  The float sum accumulates in double and rounds once to
float, so the derived bound is |r - exact| <= 1/2 ulp(exact) + n 2^-53 sum|x| (the ulp taken at |exact| plus the
accumulation bound, which covers a double sum that crossed a binade).

Shapes straddle the kernel's geometry: widths around the 256-thread row stride, heights around the grid cap
mb = 4 x SMs (rows are strided over min(h, mb) CTAs).  Every image is a view into a wider allocation whose extra
columns hold poison (NaN, +-3e38, INT_MIN, INT_MAX), so a reduction that reads past a row's width fails.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import rpg_open_remode_b200 as rmd

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
F_POISON = np.array([np.nan, 3e38, -3e38], np.float32)
I_POISON = np.array([INT_MIN, INT_MAX, INT_MIN], np.int32)


WIDTHS = [1, 31, 32, 33, 255, 256, 257, 4096]


def _mb():
    """The kernel's grid cap: 4 CTAs per SM (c_api.cu reduce_scratch)."""
    import torch
    return 4 * torch.cuda.get_device_properties(0).multi_processor_count


def _view(host, poison):
    """Upload `host` (h x w) into a (w + 3)-wide allocation with poison columns; return (view, owner)."""
    h, w = host.shape
    dtype = "float32" if host.dtype == np.float32 else "int32"
    wide = np.empty((h, w + len(poison)), host.dtype)
    wide[:, :w] = host
    wide[:, w:] = poison
    owner = rmd.DeviceImage(w + len(poison), h, dtype)
    owner.setDevData(wide)
    return rmd.DeviceImage(w, h, dtype, _view=(owner.data, owner.pitch)), owner


def _ulp32(x):
    return float(np.spacing(np.float32(min(abs(x), 3.4e38))))


def _sum_bound(x, exact):
    x = x.astype(np.float64).ravel()
    acc = x.size * 2.0 ** -53 * float(np.abs(x).sum())
    return 0.5 * _ulp32(abs(exact) + acc) + acc + abs(exact) * 2.0 ** -52


def _wrap32(v):
    return (int(v) + 2 ** 31) % 2 ** 32 - 2 ** 31


def _floats(rng, h, w, kind):
    if kind == "nonneg":
        return (rng.random((h, w)) * 2.0 ** rng.integers(-20, 20, (h, w))).astype(np.float32)
    return (rng.standard_normal((h, w)) * 2.0 ** rng.integers(-30, 30, (h, w))).astype(np.float32)


@pytest.mark.parametrize("W", WIDTHS)
def test_shapes_against_exact(W):
    rng = np.random.default_rng(W)
    red_f, red_i = rmd.ImageReducer("float32"), rmd.ImageReducer("int32")
    not_cr = total_nonneg = 0
    MB = _mb()
    for H in (1, 2, MB - 1, MB, MB + 1, 3 * MB + 7):
        for kind in ("signed", "nonneg"):
            x = _floats(rng, H, W, kind)
            v, _own = _view(x, F_POISON)
            exact = math.fsum(x.astype(np.float64).ravel())
            got = red_f.sum(v)
            assert abs(got - exact) <= _sum_bound(x, exact), (W, H, kind, got, exact)
            if kind == "nonneg":
                total_nonneg += 1
                not_cr += got != float(np.float32(exact))
            lo, hi = red_f.minMax(v)
            assert (lo, hi) == (float(x.min()), float(x.max())), (W, H)
        n = rng.integers(INT_MIN, INT_MAX, (H, W), dtype=np.int64, endpoint=True).astype(np.int32)
        v, _own = _view(n, I_POISON)
        assert red_i.sum(v) == _wrap32(int(n.astype(np.int64).sum())), (W, H)
        k = rng.choice(np.array([INT_MIN, INT_MAX, -1, 0, 5], np.int32), (H, W))
        v, _own = _view(k, I_POISON)
        for val in (INT_MIN, INT_MAX, -1, 0, 5, 6):
            assert red_i.countEqual(v, val) == int((k == val).sum()), (W, H, val)
        assert red_i.sum(v) == _wrap32(int(k.astype(np.int64).sum()))
    print(f"\nW={W}: float sum of non-negative inputs not correctly rounded in {not_cr} of {total_nonneg} images")


def test_fsum_is_exact_on_small_cases():
    """The reference itself: math.fsum equals the Fraction sum rounded to double, and the GPU sum is within the
    bound of the Fraction sum."""
    rng = np.random.default_rng(3)
    red = rmd.ImageReducer("float32")
    for (W, H) in ((1, 1), (3, 5), (33, 7), (257, 3)):
        for kind in ("signed", "nonneg"):
            x = _floats(rng, H, W, kind)
            fr = sum((Fraction(float(t)) for t in x.ravel()), Fraction(0))
            assert math.fsum(x.astype(np.float64).ravel()) == float(fr)
            v, _own = _view(x, F_POISON)
            got = red.sum(v)
            assert abs(Fraction(got) - fr) <= Fraction(_sum_bound(x, float(fr))), (W, H)


def test_float_sum_special_values():
    red = rmd.ImageReducer("float32")
    MB = _mb()
    H, W = MB + 1, 33
    base = np.full((H, W), 0.25, np.float32)
    # cancellation: +-1e30 with small terms -- inside the derived bound, whatever the order
    x = base.copy()
    x[0, 0], x[H - 1, W - 1] = 1e30, -1e30
    v, _own = _view(x, F_POISON)
    exact = math.fsum(x.astype(np.float64).ravel())
    got = red.sum(v)
    assert exact == 0.25 * (H * W - 2)
    assert abs(got - exact) <= _sum_bound(x, exact), (got, exact)
    for vals, want in (((np.inf,), np.inf), ((-np.inf,), -np.inf), ((np.inf, -np.inf), np.nan), ((np.nan,), np.nan),
                       ((3e38, 3e38), np.inf)):
        x = base.copy()
        for i, t in enumerate(vals):
            x[(i * 97) % H, (i * 13) % W] = t
        v, _own = _view(x, F_POISON)
        got = red.sum(v)
        if np.isnan(want):
            assert np.isnan(got), vals
        else:
            assert got == want, vals


def test_min_max_special_values():
    """NaN entries are ignored; an image without a non-NaN entry gives (+inf, -inf)."""
    red = rmd.ImageReducer("float32")
    MB = _mb()
    for (W, H) in ((1, 1), (33, 2), (257, MB + 1)):
        def mm(x):
            v, _own = _view(x.astype(np.float32), F_POISON)
            return red.minMax(v)
        full = lambda t: np.full((H, W), t, np.float32)   # noqa: E731
        assert mm(full(np.inf)) == (np.inf, np.inf)
        assert mm(full(-np.inf)) == (-np.inf, -np.inf)
        assert mm(full(np.nan)) == (np.inf, -np.inf)
        x = full(np.nan)
        x[H - 1, W - 1] = 2.5
        assert mm(x) == (2.5, 2.5)
        if W * H > 1:
            x = full(np.nan)
            x[0, 0], x[H - 1, W - 1] = -np.inf, np.inf
            assert mm(x) == (-np.inf, np.inf)
            x = full(1.0)
            x[0, 0] = np.inf
            assert mm(x) == (1.0, np.inf)
        lo, hi = mm(full(-0.0))
        assert lo == 0.0 and hi == 0.0
        x = full(0.0)
        x[0, 0] = -0.0
        lo, hi = mm(x)
        assert lo == 0.0 and hi == 0.0


def test_back_to_back_calls_and_errors():
    """Alternating the four operations reuses the scratch and its ticket; each result is still exact."""
    rng = np.random.default_rng(5)
    red_f, red_i = rmd.ImageReducer("float32"), rmd.ImageReducer("int32")
    MB = _mb()
    imgs = []
    for (W, H) in ((257, MB + 1), (31, 2), (4096, 3), (1, MB - 1)):
        x = _floats(rng, H, W, "nonneg")
        n = rng.integers(-3, 3, (H, W)).astype(np.int32)
        imgs.append((x, _view(x, F_POISON), n, _view(n, I_POISON)))
    for rep in range(3):
        for x, (vf, _a), n, (vi, _b) in imgs:
            exact = math.fsum(x.astype(np.float64).ravel())
            assert abs(red_f.sum(vf) - exact) <= _sum_bound(x, exact)
            assert red_i.countEqual(vi, -2) == int((n == -2).sum())
            assert red_f.minMax(vf) == (float(x.min()), float(x.max()))
            assert red_i.sum(vi) == int(n.astype(np.int64).sum())
    owner = rmd.DeviceImage(8, 8, "float32")
    for (W, H) in ((0, 8), (8, 0)):
        for dtype, ops in (("float32", (red_f.sum, red_f.minMax)), ("int32", (red_i.sum,))):
            v = rmd.DeviceImage(W, H, dtype, _view=(owner.data, owner.pitch))
            for op in ops:
                with pytest.raises(rmd.RmdError):
                    op(v)
        v = rmd.DeviceImage(W, H, "int32", _view=(owner.data, owner.pitch))
        with pytest.raises(rmd.RmdError):
            red_i.countEqual(v, 0)


def test_count_equal_beyond_2_pow_31_elements():
    """One int32 image of 2^31 + 2^16 elements (8.6 GB): the count is a 64-bit integer all the way."""
    import torch
    W, H = 65536, 32769
    need = W * H * 4
    free = torch.cuda.mem_get_info()[0]
    if free < need + (1 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    t = torch.full((H, W), 7, dtype=torch.int32, device="cuda")
    t[H - 1, W - 5:] = INT_MIN
    t[0, :3] = INT_MAX
    torch.cuda.synchronize()
    v = rmd.DeviceImage(W, H, "int32", _view=(t.data_ptr(), W * 4))
    red = rmd.ImageReducer("int32")
    assert red.countEqual(v, 7) == W * H - 8
    assert red.countEqual(v, INT_MIN) == 5
    assert red.countEqual(v, INT_MAX) == 3
    del v, t
    torch.cuda.empty_cache()
