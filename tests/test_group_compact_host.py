"""Compaction of a device group (rbk_group_compact) without a GPU: the declared and exported symbol, the copy plan of
runbookai_b200/csrc/rbk_group_plan.h compiled with g++ and replayed chunk by chunk against a numpy model of the
block-cyclic layout, and the N-API addon's compact() on a group handle against the oracle-backed stand-in of the C ABI
(tests/napi_shim/rbk_shim_group_compact.cc)."""
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from test_compact_host import check_compact_outputs, write_compact_input
from test_napi_addon import _write_inputs

DRIVER = r"""
#include <stdio.h>
#include "rbk_group_plan.h"
using namespace rbk::group_plan;
// stdin: G block chunk_blocks n_slots, then n_slots live flags.  Each member's local live ranks and per-block prefixes
// are what the compaction map kernels give the library.
int main() {
  int G;
  long long block, chunk_blocks, n;
  if (scanf("%d %lld %lld %lld", &G, &block, &chunk_blocks, &n) != 4) return 1;
  std::vector<int> live(n);
  for (long long s = 0; s < n; ++s) scanf("%d", &live[s]);
  std::vector<std::vector<int64_t>> rank(G);
  std::vector<std::vector<int>> pref(G);
  for (int e = 0; e < G; ++e) {
    const int64_t m = member_rows(G, block, n, e);
    rank[e].assign(m, -1);
    pref[e].assign((m + block - 1) / block + 1, 0);
  }
  std::vector<int64_t> cnt(G, 0);
  for (int64_t s = 0; s < n; ++s) {   // local row order within a member is global slot order
    const int e = static_cast<int>((s / block) % G);
    const int64_t l = local_row(G, block, s);
    if (l % block == 0) pref[e][l / block] = static_cast<int>(cnt[e]);
    if (live[s]) rank[e][l] = cnt[e]++;
  }
  std::vector<int64_t> block_live((n + block - 1) / block);
  for (int e = 0; e < G; ++e) pref[e].back() = static_cast<int>(cnt[e]);
  for (int64_t b = 0; b < (int64_t)block_live.size(); ++b) block_live[b] = pref[b % G][b / G + 1] - pref[b % G][b / G];
  const Plan p = make_plan(G, block, n, block_live, chunk_blocks);
  std::vector<const int64_t*> r(G);
  std::vector<const int*> bp(G);
  for (int e = 0; e < G; ++e) { r[e] = rank[e].data(); bp[e] = pref[e].data(); }
  std::vector<int64_t> map(n);
  fill_old_to_new(G, block, n, p, r, bp, map.data());
  printf("live %lld\nmap", (long long)p.n_live);
  for (int64_t v : map) printf(" %lld", (long long)v);
  printf("\n");
  for (const Chunk& c : p.chunks) {
    printf("chunk %lld %lld %lld %lld\n", (long long)c.s0, (long long)c.s1, (long long)c.d0, (long long)c.d1);
    for (int e = 0; e < G; ++e)
      printf("member %lld %lld %lld %lld\n", (long long)c.g0[e], (long long)c.gn[e], (long long)c.rank0[e],
             (long long)c.staged[e]);
    for (const Segment& s : c.segs)
      printf("seg %d %lld %d %lld %lld\n", s.src, (long long)s.src_off, s.dst, (long long)s.dst_row, (long long)s.len);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    out = tmp_path_factory.mktemp("group_plan")
    src = out / "driver.cc"
    src.write_text(DRIVER)
    exe = out / "driver"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-Wno-unused-result",
                    "-I", str(ROOT / "runbookai_b200" / "csrc"), str(src), "-o", str(exe)], check=True)
    return exe


def run_plan(exe, G, block, chunk_blocks, live):
    inp = f"{G} {block} {chunk_blocks} {len(live)}\n" + " ".join(map(str, live.astype(int))) + "\n"
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout
    chunks, n_live, old_to_new = [], None, None
    for line in out.splitlines():
        f = line.split()
        if f[0] == "live":
            n_live = int(f[1])
        elif f[0] == "map":
            old_to_new = np.array([int(v) for v in f[1:]], dtype=np.int64)
        elif f[0] == "chunk":
            chunks.append({"bounds": tuple(map(int, f[1:])), "members": [], "segs": []})
        elif f[0] == "member":
            chunks[-1]["members"].append(tuple(map(int, f[1:])))
        else:
            chunks[-1]["segs"].append(tuple(map(int, f[1:])))
    return n_live, old_to_new, chunks


def layout(G, block, n):
    """(device, local row) of every global slot below n, and each device's row count."""
    s = np.arange(n, dtype=np.int64)
    dev = (s // block) % G
    loc = (s // block // G) * block + s % block
    rows = [int((dev == d).sum()) for d in range(G)]
    return dev, loc, rows


def replay(G, block, live, chunks):
    """The move on simulated per-device arrays holding old global slots: every chunk gathers first, then applies its
    segments.  Returns the final per-device arrays."""
    n = len(live)
    dev, loc, rows = layout(G, block, n)
    store = [np.full(r, -2, dtype=np.int64) for r in rows]
    for s in range(n):
        store[dev[s]][loc[s]] = s
    glob = [dict() for _ in range(G)]                              # (device, local row) -> global slot
    for s in range(n):
        glob[dev[s]][loc[s]] = s
    last_s1 = 0
    for c in chunks:
        s0, s1, d0, d1 = c["bounds"]
        assert s0 >= last_s1 and s0 % block == 0 and s1 <= n and d1 <= s1 and d0 <= s0
        last_s1 = s1
        staging = []
        for e, (g0, gn, rank0, staged) in enumerate(c["members"]):
            part = store[e][g0:g0 + gn] if gn else np.zeros(0, np.int64)
            want = [s for s in range(s0, s1) if dev[s] == e]       # the member's share is one run of local rows
            assert list(part) == want, (e, g0, gn)
            assert rank0 == int(live[[s for s in range(n) if dev[s] == e and s < s0]].sum())
            packed = np.array([s for s in part if live[s]], dtype=np.int64)
            assert len(packed) == staged
            staging.append(packed)
        written = 0
        for src, off, dst, row, ln in c["segs"]:
            assert ln > 0 and 0 <= off and off + ln <= len(staging[src])   # only rows staged in this chunk
            for i in range(ln):
                assert glob[dst][row + i] < s1                          # never the storage of a later chunk's source
            store[dst][row:row + ln] = staging[src][off:off + ln]
            written += ln
        assert written == d1 - d0
    return store


def fresh_group(G, block, survivors):
    dev, loc, rows = layout(G, block, len(survivors))
    out = [np.full(r, -2, dtype=np.int64) for r in rows]
    for t, s in enumerate(survivors):
        out[dev[t]][loc[t]] = s
    return out


def dead_pattern(name, n, G, block, rng):
    live = np.ones(n, dtype=np.uint8)
    if name == "all":
        live[:] = 0
    elif name == "first_last":
        live[[0, n - 1]] = 0
    elif name == "blocks":                                           # whole blocks, on different devices
        for b in (1, 2, 5):
            live[b * block:(b + 1) * block] = 0
    elif name == "rounds":                                           # a whole round: every device loses a block
        live[G * block:2 * G * block] = 0
    elif name == "random40":
        live[rng.random(n) < 0.4] = 0
    elif name == "single":
        live[:] = 0
        live[n // 2 + 3] = 1
    elif name == "runs":                                             # documents of 8-40 slots
        s = 0
        while s < n:
            run = int(rng.integers(8, 41))
            if rng.random() < 0.5:
                live[s:s + run] = 0
            s += run
    elif name == "tail":                                             # only the last, partial block loses rows
        live[n - 5:] = 0
    return live


PATTERNS = ["none", "all", "first_last", "blocks", "rounds", "random40", "single", "runs", "tail"]


def test_group_compact_is_declared_and_exported(native):
    assert "rbk_group_compact" in native.SYMBOLS
    header = (ROOT / "include" / "rbk_knn.h").read_text()
    assert "rbk_status rbk_group_compact(rbk_group* grp, int64_t* old_to_new, int64_t old_to_new_len);" in header
    out = subprocess.run(["nm", "-D", "--defined-only", str(native.LIB_PATH)], capture_output=True, text=True).stdout
    assert " T rbk_group_compact\n" in out


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_plan_replays_to_a_fresh_group(planner, G, pattern):
    block = 64
    rng = np.random.default_rng(G * 100 + len(pattern))
    n = G * block * 5 + 37                                            # ends mid-block
    live = dead_pattern(pattern, n, G, block, rng)
    keep = live.astype(bool)
    survivors = np.flatnonzero(keep)
    for chunk_blocks in sorted({1, 3, G, 2 * G, 2 * G + 1}):          # multiples of a round and not
        n_live, old_to_new, chunks = run_plan(planner, G, block, chunk_blocks, live)
        assert n_live == keep.sum()
        assert (old_to_new == np.where(keep, np.cumsum(keep) - 1, -1)).all()   # the stable global rank
        if pattern == "none":
            assert chunks == []
        store = replay(G, block, live, chunks)
        want = fresh_group(G, block, survivors)
        for d in range(G):
            m = len(want[d])
            assert (store[d][:m] == want[d]).all(), (d, chunk_blocks)
        if chunks and chunk_blocks % G == 0:                         # a member's staging holds chunk_blocks / G blocks
            assert max(m[3] for c in chunks for m in c["members"]) <= chunk_blocks // G * block


def test_plan_skips_chunks_before_the_first_tombstone(planner):
    G, block = 2, 64
    n = 20 * block
    live = np.ones(n, np.uint8)
    live[9 * block + 3] = 0
    _, _, chunks = run_plan(planner, G, block, G, live)
    assert chunks[0]["bounds"][0] == 8 * block                        # the chunk holding the tombstone comes first
    # a source block crosses at most one destination block boundary: at most two segments per source block
    for c in chunks:
        assert len(c["segs"]) <= 2 * G


@pytest.fixture(scope="module")
def shim_group_compact_harness(tmp_path_factory, oracle_mod):
    """The addon harness linked against rbk_shim_group_compact.cc (built in a temporary directory)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("rbk_napi_mock_build", ROOT / "napi" / "mock" / "build.py")
    mb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mb)
    objs = mb.build_objects()
    olib = ROOT / "oracle" / "librbk_oracle.so"
    out = tmp_path_factory.mktemp("shim_group_compact")
    shim = out / "librbk_knn_shim_group_compact.so"
    mb.run(mb.CXX + ["-fPIC", "-shared", ROOT / "tests" / "napi_shim" / "rbk_shim_group_compact.cc", "-o", shim,
                     "-L", olib.parent, "-l:librbk_oracle.so", f"-Wl,-rpath,{olib.parent}"])
    exe = out / "harness_shim_group_compact"
    mb.run(["g++"] + objs + ["-o", exe, "-L", out, "-l:librbk_knn_shim_group_compact.so", f"-Wl,-rpath,{out}",
                             f"-Wl,-rpath,{olib.parent}", "-L", olib.parent, "-l:librbk_oracle.so", "-lpthread"])
    return exe


@pytest.mark.parametrize("devices", [[0], [0, 1]], ids=["one_device", "two_devices"])
def test_addon_compact_on_a_group_against_the_oracle_backed_stand_in(tmp_path, oracle_mod, shim_group_compact_harness,
                                                                      devices):
    w = _write_inputs(tmp_path, devices)
    live = write_compact_input(tmp_path, w)
    r = subprocess.run([str(shim_group_compact_harness), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    log = (tmp_path / "log.txt").read_text()
    assert "err_compact" not in log
    check_compact_outputs(tmp_path, w, oracle_mod, live)
