"""The string store's commit on the device (str_commit.cuh), held to its numpy restatement (str_commit_spec.py) byte
for byte: after every commit the published snapshot read back (oc_str_read_rows / oc_str_read_field) equals the
restated one, info() agrees, and searches equal the oracle on the restated corpus bit for bit, at several pages, with
a filter and with tombstones added before the next commit.

  - seeded random op streams over 3 fields (inserts, re-inserts in one field, deletes, insert-then-delete,
    delete-then-insert, inserts without terms, new term ids, sparse ids), several commits in a row, from an empty
    store and from a loaded 200 K-document Zipf corpus;
  - a term listed twice in one insert: the commit fails and changes nothing, and the pending ops are kept;
  - deletes from another thread while a large commit is in flight are replayed on the new snapshot, and searches
    during the commit see the old or the new snapshot;
  - a shard store (oc_str_set_global) keeps its corpus-wide N and average lengths;
  - oc_str_load_field during a commit is refused;
  - scale: the h1 corpus (1 M documents, 32 M postings) with 100 K new documents, 1 % deletes and 1 % re-inserts, and
    200 K documents inserted into an empty store in one commit."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
import str_commit_spec as spec
from oramacore_b200 import synth
from oramacore_b200._lib import OcError, check, lib
from oramacore_b200.types import StringIndexData, TextQuery
from test_gpu_topn_paths import _eq, page, ref_map

pytestmark = pytest.mark.gpu

OC_ERR_INVALID = -1   # include/oramacore_b200.h

NF = 3
PAGES = [(10, 0), (7, 5), (1000, 0)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def apply(strs, ops):
    for op in ops:
        if op[0] == "delete":
            strs.delete(op[1])
        else:
            _, f, doc, flen, pairs = op
            t = np.asarray([p[0] for p in pairs], np.uint32)
            tf = np.asarray([p[1] for p in pairs], np.uint16)
            check(lib().oc_str_insert(strs._h, f, doc, flen, len(pairs), _p(t), _p(tf)))


def assert_snapshot(strs, want):
    r = strs.read_rows()
    assert r["row_doc_ids"].tobytes() == spec.row_docs(want).tobytes()
    assert r["document_count"] == want.document_count
    for i, f in enumerate(want.fields):
        g = strs.read_field(i)
        assert g["n_terms"] == f.n_terms, i
        assert g["term_offsets"].tobytes() == f.term_offsets.astype(np.uint64).tobytes(), i
        assert g["post_row"].tobytes() == f.post_row.tobytes(), i
        assert g["post_tf"].tobytes() == f.post_tf.tobytes(), i
        assert g["post_len"].tobytes() == f.post_len.tobytes(), i
        assert g["avg_field_len"].tobytes() == np.float32(f.avg_field_len).tobytes(), (i, g["avg_field_len"], f.avg_field_len)
    info = strs.info()
    assert info["total_documents"] == want.n_rows and info["pending_postings"] == 0
    assert info["total_postings"] == sum(int(f.term_offsets[-1]) for f in want.fields)
    assert info["unique_terms_count"] == sum(f.n_terms for f in want.fields)
    return r["version"]


def doc_pairs(rng, vocab, mean=6):
    k = int(rng.poisson(mean)) + 1
    terms = np.unique(np.minimum(rng.zipf(1.4, k) - 1, vocab - 1))
    return [(int(t), int(rng.integers(1, 4))) for t in terms]


def random_ops(rng, docs, next_doc, n_ops, vocab):
    """An op stream over the committed documents `docs` (a list) and new ones from next_doc on, with gaps."""
    ops, new = [], next_doc
    for _ in range(n_ops):
        u = rng.random()
        if u < 0.45 or not docs:                           # a new document, in some of the fields
            new += int(rng.integers(1, 4))
            for f in range(NF):
                if f == 0 or rng.random() < 0.5:
                    pairs = [] if rng.random() < 0.05 else doc_pairs(rng, vocab)
                    ops.append(spec.insert(f, new, sum(p[1] for p in pairs) + int(rng.integers(0, 3)), pairs))
        elif u < 0.60:                                     # re-insert a committed document in one field
            f = int(rng.integers(0, NF))
            pairs = [] if rng.random() < 0.1 else doc_pairs(rng, vocab + 50)   # new term ids past n_terms too
            ops.append(spec.insert(f, int(rng.choice(docs)), sum(p[1] for p in pairs) + 1, pairs))
        elif u < 0.75:
            ops.append(spec.delete(int(rng.choice(docs))))
        elif u < 0.85:                                     # insert then delete
            new += 1
            ops += [spec.insert(0, new, 3, doc_pairs(rng, vocab)), spec.delete(new)]
        else:                                              # delete then insert: a new version of the document
            d = int(rng.choice(docs))
            ops += [spec.delete(d), spec.insert(int(rng.integers(0, NF)), d, 4, doc_pairs(rng, vocab))]
    return ops, new


def queries(terms):
    qs = [(f"f{f}t{t}", TextQuery.single_terms([t], field=f)) for t in terms for f in (0, 2)]
    qs.append(("multi", TextQuery.from_tokens([[(f, t, 1.0 + f) for f in range(NF)] for t in terms[:3]])))
    return qs


def check_search(ctx, orc, strs, snap, qs, dead=()):
    """Searches equal the oracle on `snap` (minus the documents `dead`, tombstoned in the store)."""
    if snap.n_rows == 0:
        return
    ix = orc.StrIndex(snap)
    docs = spec.row_docs(snap)
    nb = int(docs[-1]) + 1
    alive = np.setdiff1d(docs, np.asarray(list(dead), np.uint64))
    flt = alive[::2]
    for filt in (None, flt):
        allowed = alive if filt is None else filt
        okw = {} if filt is None and not len(dead) else dict(filter_bits=orc.make_filter_bits(allowed, nb), filter_nbits=nb)
        gkw = {} if filt is None else dict(filtered_doc_ids=orc.make_filter_bits(filt, nb), filter_nbits=nb)
        maps = [ref_map(orc, ix, q, **okw) for _, q in qs]
        for limit, offset in PAGES:
            hits = ob.search(ctx, None, strs, "fulltext", texts=[q for _, q in qs], limit=limit, offset=offset, **gkw)
            for (name, _), h, m in zip(qs, hits, maps):
                _eq(h, page(m, limit, offset), (name, limit, offset, filt is None))


def run_stream(ctx, orc, strs, snap, rng, n_commits, n_ops, vocab, next_doc):
    qs = queries([0, 1, 2, 5, 17])
    dead = []
    for _ in range(n_commits):
        ops, next_doc = random_ops(rng, spec.row_docs(snap).tolist(), next_doc, n_ops, vocab)
        ops = [spec.delete(d) for d in dead] + ops          # the tombstones of the last round are ops of this window
        apply(strs, ops[len(dead):])
        v0 = strs.info()["version"]
        st = strs.commit()
        snap = spec.commit(snap, ops)
        assert assert_snapshot(strs, snap) == v0 + 1
        assert st["rows_after"] == snap.n_rows and st["postings_after"] == sum(int(f.term_offsets[-1]) for f in snap.fields)
        check_search(ctx, orc, strs, snap, qs)
        docs = spec.row_docs(snap)
        dead = rng.choice(docs, min(len(docs), 25), replace=False).tolist() if len(docs) else []
        strs.delete(np.asarray(dead, np.uint64))
        check_search(ctx, orc, strs, snap, qs, dead)
    return snap


@pytest.mark.parametrize("seed", [1, 2])
def test_random_streams_from_empty(gpu_ctx, orc, seed):
    strs = ob.StringFieldStorage.empty(gpu_ctx, NF)
    try:
        run_stream(gpu_ctx, orc, strs, spec.empty(NF), np.random.default_rng(seed), 4, 300, 400, 0)
    finally:
        strs.close()


def zipf_corpus(n, vocab=5000, seed=7):
    fields = [synth.make_text_corpus(n, vocab, seed=seed + f, mean_len=(8.0, 3.0, 24.0)[f]).fields[0] for f in range(NF)]
    return StringIndexData(fields, n, n, None)


def test_random_streams_from_loaded_corpus(gpu_ctx, orc):
    base = zipf_corpus(200_000)
    strs = ob.StringFieldStorage(gpu_ctx, base)
    try:
        assert_snapshot(strs, StringIndexData(base.fields, base.n_rows, base.document_count, None))
        run_stream(gpu_ctx, orc, strs, base, np.random.default_rng(3), 3, 2000, 5000, 200_000)
    finally:
        strs.close()


def test_duplicate_term_fails_and_changes_nothing(gpu_ctx):
    strs = ob.StringFieldStorage.empty(gpu_ctx, NF)
    try:
        first = [spec.insert(0, d, 3, [(d % 7, 1), (9, 2)]) for d in range(50)]
        apply(strs, first)
        strs.commit()
        snap = spec.commit(spec.empty(NF), first)
        v = assert_snapshot(strs, snap)
        ops = [spec.insert(1, 60, 2, [(3, 1)]), spec.insert(2, 61, 4, [(5, 1), (8, 1), (5, 2)]), spec.delete(4)]
        apply(strs, ops)
        pending = strs.info()["pending_postings"]
        with pytest.raises(OcError) as e:
            strs.commit()
        assert "listed twice" in str(e.value)
        with pytest.raises(spec.DuplicateTerm):
            spec.commit(snap, ops)
        # the version, the snapshot and the pending ops are as before; doc 4's tombstone stays
        assert strs.read_rows()["version"] == v and strs.info()["pending_postings"] == pending
        assert strs.info()["total_documents"] == snap.n_rows - 1
        for i, f in enumerate(snap.fields):
            assert strs.read_field(i)["post_row"].tobytes() == f.post_row.tobytes()
        strs.delete(61)
        strs.commit()
        assert_snapshot(strs, spec.commit(snap, ops + [spec.delete(61)]))
    finally:
        strs.close()


def corpus_ops(data, docs, field=0, doc_ids=None):
    """Insert ops that add the documents `docs` (rows of data's field) under `doc_ids`."""
    f = data.fields[field]
    term_of = np.repeat(np.arange(f.n_terms, dtype=np.uint32), np.diff(f.term_offsets.astype(np.int64)))
    order = np.argsort(f.post_row, kind="stable")
    rows, terms, tfs = f.post_row[order], term_of[order], f.post_tf[order]
    starts = np.searchsorted(rows, np.arange(data.n_rows + 1))
    lens = np.zeros(data.n_rows, np.int64)
    lens[f.post_row] = f.post_len
    ids = docs if doc_ids is None else doc_ids
    return [spec.insert(field, int(i), int(lens[d]), list(zip(terms[starts[d]:starts[d + 1]].tolist(), tfs[starts[d]:starts[d + 1]].tolist())))
            for d, i in zip(docs.tolist(), ids.tolist())]


def test_deletes_during_a_commit_are_replayed(gpu_ctx, orc):
    base = zipf_corpus(200_000)
    strs = ob.StringFieldStorage(gpu_ctx, base)
    try:
        extra = synth.make_text_corpus(150_000, 5000, seed=99)
        ops = corpus_ops(StringIndexData(extra.fields, extra.n_rows, extra.n_rows, None), np.arange(150_000),
                         doc_ids=np.arange(150_000) + 300_000)
        apply(strs, ops)
        probe = [("p", TextQuery.single_terms([3], field=0))]
        old = ob.search(gpu_ctx, None, strs, "fulltext", texts=[probe[0][1]], limit=10)[0]
        victims = np.arange(0, 200_000, 97, dtype=np.uint64)
        seen, errs = [], []

        def committer():
            try:
                strs.commit()
            except Exception as e:   # noqa: BLE001 - reported below
                errs.append(e)

        th = threading.Thread(target=committer)
        th.start()
        for k in range(0, len(victims), 64):
            strs.delete(victims[k:k + 64])
            seen.append(ob.search(gpu_ctx, None, strs, "fulltext", texts=[probe[0][1]], limit=10)[0])
        th.join()
        assert not errs, errs
        snap = spec.commit(base, ops)
        # every victim is tombstoned in the published snapshot (or dropped by the commit when its delete came first)
        assert strs.info()["total_documents"] == snap.n_rows - len(victims)
        full = ref_map(orc, orc.StrIndex(snap), probe[0][1])[2]
        for h in seen:   # the old snapshot or the new one, less the documents deleted so far
            assert h.count <= max(old.count, full)
        strs.commit()
        assert_snapshot(strs, spec.commit(snap, [spec.delete(int(d)) for d in victims]))
    finally:
        strs.close()


def test_shard_keeps_global_values(gpu_ctx):
    base = zipf_corpus(20_000)
    strs = ob.StringFieldStorage(gpu_ctx, base)
    try:
        avgs = [11.5, 2.25, 30.0]
        strs.set_global(1_000_000, avgs)
        ops = [spec.insert(1, 50_000 + d, 5, [(d % 40, 1)]) for d in range(500)] + [spec.delete(d) for d in range(0, 300, 3)]
        apply(strs, ops)
        strs.commit()
        want = spec.commit(StringIndexData([type(f)(a, f.term_offsets, f.post_row, f.post_tf, f.post_len) for f, a in zip(base.fields, avgs)],
                                           base.n_rows, 1_000_000, None), ops, global_count=True, global_avg=True)
        r = strs.read_rows()
        assert r["document_count"] == 1_000_000
        assert_snapshot(strs, want)
    finally:
        strs.close()


def test_load_field_during_a_commit_is_refused(gpu_ctx):
    strs = ob.StringFieldStorage.empty(gpu_ctx, 1)
    try:
        extra = synth.make_text_corpus(200_000, 5000, seed=5)
        ops = corpus_ops(extra, np.arange(200_000))
        apply(strs, ops)
        th = threading.Thread(target=strs.commit)
        zero = np.zeros(1, np.uint64)
        refused = False
        th.start()
        while th.is_alive() and not refused:
            # an empty field 0: a no-op before the commit starts (the store has no committed postings)
            rc = lib().oc_str_load_field(strs._h, 0, 0.0, 0, _p(zero), None, None, None, None)
            assert rc in (0, OC_ERR_INVALID), rc
            refused = rc == OC_ERR_INVALID
        th.join()
        assert refused, "the commit ended before a load could overlap it"
        assert_snapshot(strs, spec.commit(spec.empty(1), ops))
    finally:
        strs.close()


def test_scale_h1_corpus(gpu_ctx):
    rng = np.random.default_rng(11)
    n = 1_000_000
    base = synth.make_text_corpus(n, 200_000)
    assert int(base.fields[0].term_offsets[-1]) > 30_000_000
    strs = ob.StringFieldStorage(gpu_ctx, base)
    try:
        extra = synth.make_text_corpus(100_000, 200_000, seed=12)
        ops = corpus_ops(extra, np.arange(100_000), doc_ids=np.arange(100_000) + n)
        ops += [spec.delete(int(d)) for d in rng.choice(n, n // 100, replace=False)]
        ops += corpus_ops(extra, rng.choice(100_000, n // 100, replace=False), doc_ids=rng.choice(n, n // 100, replace=False))
        apply(strs, ops)
        st = strs.commit()
        assert_snapshot(strs, spec.commit(base, ops))
        assert st["postings_before"] == int(base.fields[0].term_offsets[-1]) and st["device_ms"] > 0
    finally:
        strs.close()


def test_scale_200k_documents_into_an_empty_store(gpu_ctx):
    data = synth.make_text_corpus(200_000, 50_000, seed=21)
    strs = ob.StringFieldStorage.empty(gpu_ctx, 1)
    try:
        ops = corpus_ops(data, np.arange(200_000))
        apply(strs, ops)
        st = strs.commit()
        assert st["pending_postings"] == int(data.fields[0].term_offsets[-1]) > 5_000_000
        want = spec.commit(spec.empty(1), ops)
        assert_snapshot(strs, want)
        f = data.fields[0]   # the same CSR as the bulk corpus
        assert want.fields[0].post_row.tobytes() == f.post_row.tobytes()
        assert want.fields[0].term_offsets.tobytes() == f.term_offsets.tobytes()
    finally:
        strs.close()
