"""CPU suite: embedding widths outside 8-2048.

- The C oracle (rbk_oracle.c) against the pure-Python restatement (oracle/pyref.py) at the widths the GPU suite
  (test_gpu_widths.py) checks the engine at: the oracle is the reference there, so it is checked first.
- The width limit of the C ABI: rbk_index_create_ex and rbk_group_create reject 0 and RBK_MAX_DIM + 1 with RBK_EINVAL
  before looking for a device, and accept RBK_MAX_DIM itself (RBK_ECUDA without a device).
- The oracle-backed stand-in of the ABI (tests/napi_shim/rbk_shim.cc) keeps the same limit."""
import ctypes as C

import numpy as np
import pytest

from conftest import HAS_CUDA
from test_napi_addon import _build_shim

MAX_DIM = 1 << 20
WIDTHS = (1, 2, 3, 5, 7, 2049, 3072, 4095, 4096, 8192, 16384, 65536)


def test_oracle_cosine_matches_python_at_every_width(oracle_mod):
    from oracle import pyref
    rng = np.random.default_rng(12)
    for d in WIDTHS + (MAX_DIM,):
        for t in range(1 if d == MAX_DIM else 6):
            a, b = rng.standard_normal(d), rng.standard_normal(d)
            if t == 1:
                a, b = np.abs(a), np.abs(b)                   # all-positive: nothing cancels in the dot chain
            if t == 2:
                a = a * 2.0 ** -500                           # norms that underflow
            assert oracle_mod.cosine(a, b) == pyref.cosine_similarity(a.tolist(), b.tolist()), (d, t)


@pytest.mark.parametrize("d", [1, 2, 3, 5, 7, 2049, 4095, 16384])
def test_oracle_search_matches_python_at_every_width(oracle_mod, d):
    """find_most_similar and the thresholded scan of pyref against the oracle's f64 and bf16 searches: duplicates
    (ties by slot), a zero row and, at d = 1, every row tied at +-1."""
    from oracle import pyref
    from runbookai_b200 import synth
    rng = np.random.default_rng(d)
    n = 40 if d > 1000 else 300
    rows = rng.standard_normal((n, d))
    rows[5] = 0.0
    rows[9] = rows[3]
    rows[n - 1] = rows[3]
    q = rng.standard_normal(d)
    bits = synth.f32_to_bf16_bits(rows.astype(np.float32))
    rows_bf16 = synth.bf16_bits_to_f32(bits).astype(np.float64)
    for corpus, stored in ((rows, rows), (bits, rows_bf16)):
        emb = list(enumerate(stored.tolist()))
        want = pyref.find_most_similar(q.tolist(), emb, n)
        s, v = oracle_mod.search(corpus, q, n, None)
        assert s.tolist() == [i for i, _ in want] and v.tolist() == [x for _, x in want]
        want = pyref.vector_scan(q.tolist(), emb, top_k=n, min_score=0.01)
        s, v = oracle_mod.search(corpus, q, 2 * n, 0.01)
        assert s.tolist() == [i for i, _ in want] and v.tolist() == [x for _, x in want]
    if d == 1:
        s, v = oracle_mod.search(rows, q, n, None)
        assert set(np.abs(v)) == {1.0} and len(s) == n - 1
        assert (np.diff(s[v == v[0]]) > 0).all()


def _create_calls(lib):
    vp = C.c_void_p
    lib.rbk_index_create_ex.argtypes = [C.c_int32, C.c_int32, C.c_int64, C.c_uint32, C.POINTER(vp)]
    lib.rbk_group_create.argtypes = [C.c_int32, vp, C.c_int32, C.c_int64, C.c_uint32, C.POINTER(vp)]
    lib.rbk_index_destroy.argtypes = [vp]
    lib.rbk_group_destroy.argtypes = [vp]
    lib.rbk_last_error.restype = C.c_char_p
    dev = np.zeros(1, dtype=np.int32)

    def index(dim):
        h = vp()
        st = lib.rbk_index_create_ex(dim, 0, 0, 0, C.byref(h))
        if h.value:
            lib.rbk_index_destroy(h)
        return st, lib.rbk_last_error().decode()

    def group(dim):
        h = vp()
        st = lib.rbk_group_create(dim, dev.ctypes.data_as(vp), 1, 0, 0, C.byref(h))
        if h.value:
            lib.rbk_group_destroy(h)
        return st, lib.rbk_last_error().decode()

    return index, group


def test_abi_width_limit(native):
    """0 and RBK_MAX_DIM + 1 are arguments out of range whatever the machine; RBK_MAX_DIM passes the check and, without
    a device, fails for want of one."""
    index, group = _create_calls(native.lib)
    for create in (index, group):
        for dim in (0, -1, MAX_DIM + 1, 1 << 30):
            st, msg = create(dim)
            assert st == native.RBK_EINVAL and "dim out of range" in msg, (create.__name__, dim, st, msg)
        if not HAS_CUDA:
            st, msg = create(MAX_DIM)
            assert st == native.RBK_ECUDA and "no CUDA device" in msg, (create.__name__, st, msg)


def test_shim_width_limit(native):
    """The oracle-backed stand-in rejects the widths the library rejects and accepts the ones it accepts."""
    _build_shim()
    from conftest import ROOT
    shim = C.CDLL(str(ROOT / "tests" / "napi_shim" / "_build" / "librbk_knn_shim.so"))
    index, group = _create_calls(shim)
    for create in (index, group):
        for dim in (0, MAX_DIM + 1):
            assert create(dim)[0] == native.RBK_EINVAL, (create.__name__, dim)
        for dim in (1, 4095, MAX_DIM):
            assert create(dim)[0] == native.RBK_OK, (create.__name__, dim)
