"""Changing a float64-backed index's storage tier without a GPU: the declared and exported symbols, the flag arithmetic of
`Index.set_tier` / `Group.set_tier` down to rbk_index_set_tier / rbk_group_set_tier through a recording stand-in of the
library, and `VectorStore.set_tier` with its tier properties on a CPU index stand-in."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from common import HashEmbedder, OracleIndex
from conftest import ROOT

KEEP, HOST, F16 = 1, 2, 16


def test_header_declares_and_library_exports_the_entry_points(native):
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    for name, decl in (("rbk_index_flags", "uint32_t rbk_index_flags(const rbk_index* idx);"),
                       ("rbk_index_set_tier", "rbk_status rbk_index_set_tier(rbk_index* idx, uint32_t flags);"),
                       ("rbk_group_set_tier", "rbk_status rbk_group_set_tier(rbk_group* grp, uint32_t flags);")):
        assert name in native.SYMBOLS and decl in header
    assert "fixed for the index's life" not in header
    out = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True).stdout
    for name in ("rbk_index_flags", "rbk_index_set_tier", "rbk_group_set_tier"):
        assert f" T {name}\n" in out
    assert native.lib.rbk_abi_version() == 2


def test_null_handles(native):
    assert native.lib.rbk_index_flags(None) == 0
    assert native.lib.rbk_index_set_tier(None, KEEP) == native.RBK_EINVAL
    assert native.lib.rbk_group_set_tier(None, KEEP) == native.RBK_EINVAL


class TierLib:
    """Stands in for librbk_knn.so: creates handles, records every set_tier call and keeps each handle's flags."""

    def __init__(self):
        self.flags = {}
        self.calls = []

    def rbk_index_create_ex(self, dim, device, hint, flags, out):
        h = 0x1000 + len(self.flags)
        self.flags[h] = flags
        out._obj.value = h
        return 0

    def rbk_group_create(self, dim, devs, n, hint, flags, out):
        return self.rbk_index_create_ex(dim, 0, hint, flags, out)

    def rbk_group_member(self, g, i):
        return g.value

    def rbk_index_flags(self, h):
        return self.flags[h.value if isinstance(h, C.c_void_p) else h]

    def _set(self, kind, h, flags):
        h = h.value if isinstance(h, C.c_void_p) else h
        self.calls.append((kind, flags))
        if not flags & KEEP:
            return 1
        self.flags[h] = flags
        return 0

    def rbk_index_set_tier(self, h, flags):
        return self._set("index", h, flags)

    def rbk_group_set_tier(self, h, flags):
        return self._set("group", h, flags)

    def rbk_last_error(self):
        return b"RBK_INDEX_F64_ON_HOST requires RBK_INDEX_KEEP_F64"

    def rbk_index_destroy(self, h):
        pass

    rbk_group_destroy = rbk_index_destroy


@pytest.fixture
def tierlib(native, monkeypatch):
    lib = TierLib()
    monkeypatch.setattr(native, "lib", lib)
    return lib


@pytest.mark.parametrize("kind", ["index", "group"])
def test_set_tier_flag_arithmetic(native, tierlib, kind):
    ix = native.Index(64, keep_f64=True) if kind == "index" else native.Group(64, [0], keep_f64=True)
    assert ix.flags == KEEP
    ix.set_tier(f64_on_host=True)
    assert ix.flags == KEEP | HOST
    ix.set_tier(scan_f16=True)                        # None keeps the placement
    assert ix.flags == KEEP | HOST | F16
    ix.set_tier(f64_on_host=False)
    assert ix.flags == KEEP | F16
    ix.set_tier()                                     # nothing asked: the current flags, which the library accepts
    ix.set_tier(f64_on_host=np.bool_(True), scan_f16=False)
    assert ix.flags == KEEP | HOST
    assert tierlib.calls == [(kind, KEEP | HOST), (kind, KEEP | HOST | F16), (kind, KEEP | F16), (kind, KEEP | F16),
                             (kind, KEEP | HOST)]
    ix.close()


def test_set_tier_argument_checks(native, tierlib):
    ix = native.Index(64, keep_f64=True)
    for bad in ({"f64_on_host": 1}, {"scan_f16": "yes"}, {"f64_on_host": None, "scan_f16": 0.0}):
        with pytest.raises(TypeError, match="must be a bool or None"):
            ix.set_tier(**bad)
    with pytest.raises(TypeError):
        ix.set_tier(True)                             # keyword-only
    assert tierlib.calls == []
    plain = native.Index(64)
    with pytest.raises(native.RbkError, match="requires RBK_INDEX_KEEP_F64") as e:
        plain.set_tier(f64_on_host=True)              # KEEP_F64 is not added: the library refuses
    assert e.value.status == native.RBK_EINVAL and tierlib.calls == [("index", HOST)]
    ix.close()                                        # while the stand-in is still the library
    plain.close()


class TierOracleIndex(OracleIndex):
    """The CPU index stand-in with the tier surface of _native.Index: flags and set_tier (the rows do not change, as
    the answers of the real index do not)."""

    def __init__(self, dim, device=0, flags=KEEP):
        super().__init__(dim, device)
        self.flags = flags
        self.tier_calls = []

    def set_tier(self, *, f64_on_host=None, scan_f16=None):
        self.tier_calls.append((f64_on_host, scan_f16))
        if f64_on_host is not None:
            self.flags = self.flags | HOST if f64_on_host else self.flags & ~HOST
        if scan_f16 is not None:
            self.flags = self.flags | F16 if scan_f16 else self.flags & ~F16


@pytest.fixture
def hash_embedder():
    from runbookai_b200 import embedder
    embedder.configure(HashEmbedder(64))
    yield
    embedder.reset()


def _chunks(doc, n):
    words = ["redis", "pool", "postgres", "failover", "kubernetes", "pod", "gateway", "tls", "latency", "oom"]
    return [{"chunk": {"id": f"{doc}_{i}", "documentId": doc, "sectionTitle": "S",
                       "content": " ".join(words[(i + j) % len(words)] for j in range(4)) + f" {i}"},
             "documentTitle": doc.upper(), "type": "runbook", "services": ["api"]} for i in range(n)]


def _answers(vs):
    return [[(c.id, c.score) for c in vs.search(q, {"topK": 5, "minScore": 0.1})]
            for q in ("redis pool", "postgres failover", "gateway tls latency")]


def test_vector_store_set_tier_on_a_shared_index(tmp_path, monkeypatch, hash_embedder):
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    monkeypatch.delenv("RUNBOOK_KNN_F64_ON_HOST", raising=False)
    monkeypatch.delenv("RUNBOOK_KNN_SCAN_F16", raising=False)
    made = []

    def factory(dim, dev):
        made.append(TierOracleIndex(dim, dev))
        return made[-1]

    path = str(tmp_path / "vectors.db")
    a = VectorStore(path, index_factory=factory, shared=True)
    assert (a.f64_on_host, a.scan_f16) == (False, False)
    a.set_tier(scan_f16=True)                         # no index yet: the request is this instance's
    assert (a.f64_on_host, a.scan_f16) == (False, True) and made == []
    a.add_chunks(_chunks("d0", 12))
    ix = a._index
    assert ix is made[0]
    ix.flags = KEEP                                   # the index reports its own tier, whatever was asked
    assert (a.f64_on_host, a.scan_f16) == (False, False)
    b = VectorStore(path, index_factory=factory, shared=True, f64_on_host=True, scan_f16=True)
    assert b._index is ix and (b.f64_on_host, b.scan_f16) == (False, False)
    want = _answers(a)
    b.set_tier(f64_on_host=True, scan_f16=True)
    assert ix.tier_calls == [(True, True)]
    assert (a.f64_on_host, a.scan_f16, b.f64_on_host, b.scan_f16) == (True, True, True, True)
    a.set_tier(scan_f16=False)
    assert ix.tier_calls[-1] == (None, False) and (b.f64_on_host, b.scan_f16) == (True, False)
    assert _answers(a) == want and _answers(b) == want
    with pytest.raises(TypeError, match="must be a bool or None"):
        a.set_tier(f64_on_host="no")
    assert len(ix.tier_calls) == 2
    b.close()
    a.close()


def test_vector_store_set_tier_needs_an_index_that_has_tiers(tmp_path, monkeypatch, hash_embedder):
    from runbookai_b200.vector_store import VectorStore
    monkeypatch.setenv("RUNBOOK_KNN_SIDECAR", "0")
    vs = VectorStore(str(tmp_path / "v.db"), index_factory=lambda d, dev: OracleIndex(d))
    vs.add_chunks(_chunks("d0", 4))
    assert vs.f64_on_host in (False, True)            # an index without flags: the request stands
    with pytest.raises(NotImplementedError):
        vs.set_tier(f64_on_host=True)
    vs.close()


def test_addon_set_tier_against_a_library_without_it(tmp_path, oracle_mod):
    """An ABI-2 library built before tier changes (here: the oracle-backed stand-in of the C ABI) still loads the addon
    and runs every other method; `tier` and `setTier` throw instead of the module failing to load."""
    from test_napi_addon import _build_shim, _check_outputs, _write_inputs
    exe = _build_shim()
    w = _write_inputs(tmp_path, [])
    (tmp_path / "set_tier.txt").write_text("1 1\n")
    r = subprocess.run([str(exe), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    log = dict(line.split(" ", 1) for line in (tmp_path / "log.txt").read_text().strip().splitlines())
    assert "no tier change" in log["err_set_tier"] and "tier_after" not in log
    _check_outputs(tmp_path, w, oracle_mod)
