"""oc_emb_compact without a device: the symbol and the struct layout, the wrapper's argument handling, and a numpy
restatement of what the device code computes — the destination map (row minus the dead rows below it, from a per-word
popcount and two exclusive scans) and the window schedule that makes the move safe in place."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCAN_WORDS = 1024   # COMPACT_SCAN_WORDS (emb_compact.cuh)


def test_symbol_and_struct_layout(tmp_path):
    ob.build()
    L = ob.lib()
    assert hasattr(L, "oc_emb_compact") and "oc_emb_compact" in _lib.EXPORTED_SYMBOLS
    # the header's struct as a C compiler lays it out against the ctypes mirror
    src = tmp_path / "layout.c"
    fields = [n for n, _ in _lib.EmbCompact._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "oramacore_b200.h"\nint main(void) {\n'
                   '  printf("%zu", sizeof(oc_emb_compact_t));\n'
                   + "".join(f'  printf(" %zu", offsetof(oc_emb_compact_t, {f}));\n' for f in fields)
                   + '  printf(" %u", OC_EMB_COMPACT_SHRINK);\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[0] == C.sizeof(_lib.EmbCompact)
    assert got[1:-1] == [getattr(_lib.EmbCompact, f).offset for f in fields]
    assert got[-1] == _lib.OC_EMB_COMPACT_SHRINK


def test_refusals_need_no_device():
    L = ob.lib()
    st = _lib.EmbCompact()
    assert L.oc_emb_compact(None, 0, C.byref(st)) == -1            # OC_ERR_INVALID
    assert "NULL" in L.oc_last_error().decode()
    with pytest.raises(ob.OcError) as e:
        _lib.check(L.oc_emb_compact(None, 0, None))
    assert e.value.code == -1


def test_no_store_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    # a store hangs off a context, and a context needs a device: like every device entry point, compaction is out of
    # reach without one (OC_ERR_CUDA from oc_init, no CPU path)
    with pytest.raises(ob.OcError) as e:
        ob.Context(0)
    assert e.value.code == -2


def test_wrapper_passes_the_flag_and_returns_the_stats(monkeypatch):
    calls = []

    class FakeLib:
        def oc_emb_compact(self, h, flags, out):
            calls.append((h, flags))
            st = C.cast(out, C.POINTER(_lib.EmbCompact)).contents
            st.rows_before, st.rows_after, st.rows_moved, st.device_ms = 10, 7, 5, 0.5
            return 0

    from oramacore_b200 import engine
    monkeypatch.setattr(engine, "lib", lambda: FakeLib())
    emb = ob.EmbeddingFieldStorage.__new__(ob.EmbeddingFieldStorage)
    emb._h = C.c_void_p(1234)
    st = emb.compact()
    assert calls[-1][1] == 0
    assert set(st) == {n for n, _ in _lib.EmbCompact._fields_}
    assert (st["rows_before"], st["rows_after"], st["rows_moved"], st["device_ms"]) == (10, 7, 5, 0.5)
    emb.compact(shrink=True)
    assert calls[-1][1] == _lib.OC_EMB_COMPACT_SHRINK
    emb._h = C.c_void_p()


# ---- the device algorithm, restated


def _dead_below_scanned(dead_mask):
    """dead rows below every row, the way the kernels derive it: popcount per 32-row word, exclusive scan of the words of
    each scan block, exclusive scan of the block totals, popcount of the word's bits below the row."""
    n = dead_mask.shape[0]
    n_words = (n + 31) // 32
    padded = np.zeros(n_words * 32, bool)
    padded[:n] = dead_mask
    per_word = padded.reshape(n_words, 32).sum(1).astype(np.uint32)
    n_blocks = (n_words + SCAN_WORDS - 1) // SCAN_WORDS
    word_pre = np.zeros(n_words, np.uint32)
    block_tot = np.zeros(n_blocks, np.uint32)
    for b in range(n_blocks):
        w = per_word[b * SCAN_WORDS:(b + 1) * SCAN_WORDS]
        word_pre[b * SCAN_WORDS:b * SCAN_WORDS + w.shape[0]] = np.cumsum(w) - w
        block_tot[b] = w.sum()
    block_pre = np.cumsum(block_tot) - block_tot
    in_word = padded.reshape(n_words, 32).cumsum(1) - padded.reshape(n_words, 32)
    r = np.arange(n)
    return block_pre[(r >> 5) // SCAN_WORDS] + word_pre[r >> 5] + in_word.reshape(-1)[:n]


def _windows(n, dead_sorted, w_rows):
    """(a, b, dst, live) of every window the host issues, in order (oc_emb_compact)."""
    out = []
    if dead_sorted.shape[0] == 0:
        return out
    a = int(dead_sorted[0])
    while a < n:
        b = min(n, a + w_rows)
        below = int(np.searchsorted(dead_sorted, a))
        live = (b - a) - (int(np.searchsorted(dead_sorted, b)) - below)
        if live:
            out.append((a, b, a - below, live))
        a += w_rows
    return out


def _dead_sets(rng, n):
    yield rng.random(n) < 0.1
    yield rng.random(n) < 0.5
    yield rng.random(n) < 0.97
    m = np.zeros(n, bool); m[n // 3:n // 2] = True; yield m          # a contiguous run
    m = np.zeros(n, bool); m[:n // 4] = True; yield m                 # the first rows
    m = np.zeros(n, bool); m[-(n // 4):] = True; yield m              # the last rows
    m = np.ones(n, bool); m[n // 2] = False; yield m                  # all but one
    yield np.ones(n, bool)
    m = np.zeros(n, bool); m[n - 1] = True; yield m


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 32 * SCAN_WORDS - 1, 32 * SCAN_WORDS + 5, 3 * 32 * SCAN_WORDS + 77])
def test_destination_map(n):
    rng = np.random.default_rng(n)
    for dead in _dead_sets(rng, n):
        below = _dead_below_scanned(dead)
        assert np.array_equal(below, np.cumsum(dead) - dead)
        live = np.flatnonzero(~dead)
        # order-preserving and dense: the live rows land on 0 .. n_live - 1 in their order
        assert np.array_equal(live - below[live], np.arange(live.shape[0]))


@pytest.mark.parametrize("n,w_rows", [(1000, 1), (1000, 7), (1000, 256), (5000, 999), (5000, 5000), (5000, 100000)])
def test_window_schedule_is_safe_in_place(n, w_rows):
    rng = np.random.default_rng(n + w_rows)
    for dead in _dead_sets(rng, n):
        dead_sorted = np.flatnonzero(dead)
        store = np.arange(n)                     # the array being compacted: row r holds r
        consumed = int(dead_sorted[0]) if dead_sorted.shape[0] else n     # source rows below this were read (or never move)
        for a, b, dst, live in _windows(n, dead_sorted, w_rows):
            assert a >= consumed                 # windows ascend and do not overlap
            staged = store[a:b][~dead[a:b]].copy()        # the gather: this window's live rows, in order
            assert staged.shape[0] == live
            # the store range lies at or below the window it came from and never reaches an unread source row
            assert dst <= a and dst + live <= b
            store[dst:dst + live] = staged
            consumed = b
        n_live = int((~dead).sum())
        expect = np.flatnonzero(~dead)
        assert np.array_equal(store[:n_live], expect)
        # rows below the first dead row are not touched by any window
        first = int(dead_sorted[0]) if dead_sorted.shape[0] else n
        assert all(dst >= first for _, _, dst, _ in _windows(n, dead_sorted, w_rows))


def test_doc_rows_remap_matches_the_map():
    rng = np.random.default_rng(3)
    n = 4000
    dead = rng.random(n) < 0.3
    dead_sorted = np.flatnonzero(dead)
    live = np.flatnonzero(~dead)
    assert np.array_equal(live - np.searchsorted(dead_sorted, live), np.arange(live.shape[0]))
