"""The numeric contract (include/kjb_numeric.h) against libm / numpy: stated error bounds, f16 conversions exact."""
import ctypes as C, os, subprocess, numpy as np, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = r'''
#include "kjb_numeric.h"
#define E(name, expr) void name(const float* a, const float* b, float* o, int n) { for (int i = 0; i < n; ++i) o[i] = expr; }
E(t_sin, kjb_sin(a[i])) E(t_cos, kjb_cos(a[i])) E(t_exp2, kjb_exp2(a[i])) E(t_log2, kjb_log2(a[i])) E(t_pow, kjb_pow(a[i], b[i]))
E(t_atan, kjb_atan(a[i])) E(t_atan2, kjb_atan2(a[i], b[i])) E(t_acos, kjb_acos(a[i])) E(t_min, kjb_min(a[i], b[i])) E(t_max, kjb_max(a[i], b[i]))
int t_div_int_const(void) {   /* number of (numerator, divisor) pairs where the 3-instruction form differs from IEEE division: must be 0 */
    const float ds[] = {127.0f, 255.0f, 1023.0f, 2047.0f, 32767.0f, 65535.0f}; int bad = 0;
    for (int k = 0; k < 6; ++k) for (int i = -70000; i <= 70000; ++i) { const float x = (float)i; const float a = kjb_div_int_const(x, ds[k], 1.0f / ds[k]), b = x / ds[k]; bad += kjb_f2u(a) != kjb_f2u(b); }
    return bad;
}
void t_f2h(const float* a, unsigned* o, int n) { for (int i = 0; i < n; ++i) o[i] = kjb_f32_to_f16(a[i]); }
void t_h2f(const unsigned* a, float* o, int n) { for (int i = 0; i < n; ++i) o[i] = kjb_f16_to_f32(a[i]); }
void t_cvt(const float* a, int* o, unsigned* u, int n) { for (int i = 0; i < n; ++i) { o[i] = kjb_cvt_i32(a[i]); u[i] = kjb_cvt_u32(a[i]); } }
'''


@pytest.fixture(scope="module")
def num(tmp_path_factory):
    d = tmp_path_factory.mktemp("num")
    (d / "n.c").write_text(SRC)
    so = d / "n.so"
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"), str(d / "n.c"), "-o", str(so), "-lm"])
    return C.CDLL(str(so))


def _call(lib, name, a, b=None):
    a = np.ascontiguousarray(a, np.float32); b = np.ascontiguousarray(b if b is not None else a, np.float32); o = np.empty_like(a)
    getattr(lib, name)(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p), C.c_int(a.size))
    return o


def test_trig(num):
    x = np.random.RandomState(0).uniform(-300, 300, 200000).astype(np.float32)
    assert np.abs(_call(num, "t_sin", x) - np.sin(x.astype(np.float64))).max() < 2e-7
    assert np.abs(_call(num, "t_cos", x) - np.cos(x.astype(np.float64))).max() < 2e-7
    a = np.random.RandomState(1).uniform(-50, 50, 100000).astype(np.float32)
    assert np.abs(_call(num, "t_atan", a) - np.arctan(a.astype(np.float64))).max() < 4e-7
    c = np.random.RandomState(2).uniform(-1, 1, 100000).astype(np.float32)
    assert np.abs(_call(num, "t_acos", c) - np.arccos(c.astype(np.float64))).max() < 1e-6


def test_exp_log_pow(num):
    x = np.random.RandomState(3).uniform(-125, 127, 200000).astype(np.float32)
    r = np.exp2(x.astype(np.float64))
    assert (np.abs(_call(num, "t_exp2", x) - r) / r).max() < 3e-7
    z = np.exp2(np.random.RandomState(4).uniform(-40, 40, 200000)).astype(np.float32)
    assert np.abs(_call(num, "t_log2", z) - np.log2(z.astype(np.float64))).max() < 4e-6
    b = np.random.RandomState(5).uniform(1e-3, 4, 100000).astype(np.float32); e = np.random.RandomState(6).uniform(0, 8, 100000).astype(np.float32)
    r = np.power(b.astype(np.float64), e.astype(np.float64))
    assert (np.abs(_call(num, "t_pow", b, e) - r) / r).max() < 2e-5
    assert _call(num, "t_pow", [0.0], [0.5])[0] == 0.0 and _call(num, "t_exp2", [0.0])[0] == 1.0 and _call(num, "t_log2", [1.0])[0] == 0.0


def test_minmax_nan_semantics(num):
    nan = np.float32(np.nan)
    assert _call(num, "t_max", [0.0], [nan])[0] == 0.0 and _call(num, "t_max", [nan], [0.0])[0] == 0.0
    assert _call(num, "t_min", [1.0], [nan])[0] == 1.0 and _call(num, "t_min", [nan], [1.0])[0] == 1.0


def test_f16_nan_is_canonical(num):
    """Every f32 NaN, either sign and any payload, stores as 0x7e00: the GPU's 0/0 is +NaN and x86's is -NaN, and a NaN the
    shaders produce (filter_history.hlsl:44 when every luma weight is 0) must be stored the same by the kernels and the oracle."""
    rng = np.random.RandomState(9)
    bits = np.concatenate([np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fffffff, 0xffffffff], np.uint32),
                           (0x7f800001 + rng.randint(0, 0x7fffff, 1000)).astype(np.uint32) | (rng.randint(0, 2, 1000).astype(np.uint32) << 31)])
    x = bits.view(np.float32)
    out = np.empty(x.size, np.uint32)
    num.t_f2h(x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_int(x.size))
    assert (out == 0x7e00).all()


def test_f16_exhaustive_and_random(num):
    h = np.arange(65536, dtype=np.uint32); o = np.empty(65536, np.float32)
    num.t_h2f(h.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p), C.c_int(65536))
    ref = h.astype(np.uint16).view(np.float16).astype(np.float32)
    ok = np.isnan(ref) | (o.view(np.uint32) == ref.view(np.uint32))
    assert ok.all()
    x = np.random.RandomState(7).uniform(-70000, 70000, 400000).astype(np.float32)
    x = np.concatenate([x, (np.random.RandomState(8).randn(200000) * 1e-5).astype(np.float32), np.array([0.0, -0.0, 65504.0, 65519.9, 65520.0, 1e-8, 5.96e-8, 2.98e-8], np.float32)])
    out = np.empty(x.size, np.uint32)
    num.t_f2h(x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_int(x.size))
    with np.errstate(over="ignore"):
        assert (out == x.astype(np.float16).view(np.uint16)).all()


def test_saturating_conversions(num):
    x = np.array([0.0, -0.5, 1.9, -1.9, 3e9, -3e9, 5e9, np.nan, 2147483520.0], np.float32)
    i = np.empty(x.size, np.int32); u = np.empty(x.size, np.uint32)
    num.t_cvt(x.ctypes.data_as(C.c_void_p), i.ctypes.data_as(C.c_void_p), u.ctypes.data_as(C.c_void_p), C.c_int(x.size))
    assert i.tolist() == [0, 0, 1, -1, 2147483647, -2147483648, 2147483647, 0, 2147483520]
    assert u.tolist() == [0, 0, 1, 0, 3000000000, 0, 4294967295, 0, 2147483520]


def test_integer_over_constant_division_is_ieee_exact(num):
    """kjb_div_int_const (texel decode on the device) == the `/` the oracle writes, for every numerator any texel format can produce"""
    assert num.t_div_int_const() == 0


def test_min_max_order_signed_zeros_and_drop_nans(num):
    """IEEE 754-2019 minimumNumber / maximumNumber — what FMNMX does on sm_90a (tools/probe_minmax.cu)"""
    u = lambda *w: np.array(w, np.uint32).view(np.float32)
    a = u(0x00000000, 0x80000000, 0x00000000, 0x80000000, 0x7fc00000, 0x3f800000, 0xffc12345, 0x80000000, 0x7fc00000, 0x00000001, 0x80000001)
    b = u(0x80000000, 0x00000000, 0x00000000, 0x80000000, 0x3f800000, 0x7fc00000, 0x80000000, 0xffc12345, 0xffc12345, 0x80000001, 0x00000001)
    mn = u(0x80000000, 0x80000000, 0x00000000, 0x80000000, 0x3f800000, 0x3f800000, 0x80000000, 0x80000000, 0x7fffffff, 0x80000001, 0x80000001)   # as printed by the H100
    mx = u(0x00000000, 0x00000000, 0x00000000, 0x80000000, 0x3f800000, 0x3f800000, 0x80000000, 0x80000000, 0x7fffffff, 0x00000001, 0x00000001)
    assert np.array_equal(_call(num, "t_min", a, b).view(np.uint32), mn.view(np.uint32))
    assert np.array_equal(_call(num, "t_max", a, b).view(np.uint32), mx.view(np.uint32))
    x = np.random.RandomState(3).standard_normal(100000).astype(np.float32); y = np.random.RandomState(4).standard_normal(100000).astype(np.float32)
    assert np.array_equal(_call(num, "t_min", x, y), np.minimum(x, y)) and np.array_equal(_call(num, "t_max", x, y), np.maximum(x, y))
