"""torchrun worker for oc_str_sync_global over NCCL: every rank loads its shard without df tables, commits, syncs, and
must then hold the whole corpus's df table and average, and answer sharded fulltext batches byte for byte as the
unsharded store does.
Run: python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/sharded_sync_worker.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import torch.distributed as dist
    import oramacore_b200 as ob
    from oramacore_b200 import synth
    from oramacore_b200.engine import TokenScoreContext, TokenScoreParams
    from oramacore_b200.sharding import shard_range, shard_string_index
    from oramacore_b200.types import MODE_FULLTEXT

    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    ctx = ob.Context(lr)
    uid = [ob.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(world, rank, uid[0])

    n, vocab, B = 60000, 3000, 16
    data = synth.make_text_corpus(n, vocab, seed=43)
    texts = synth.make_text_queries(vocab, B, seed=44)
    sd, _ = shard_string_index(data, *shard_range(n, rank, world))
    strs = ob.StringFieldStorage(ctx, sd)          # no df table
    strs.commit()
    st = strs.sync_global()
    f = data.fields[0]
    assert st["rows_global"] == n, st
    assert np.array_equal(strs.read_global_df(0), np.diff(f.term_offsets.astype(np.int64)).astype(np.uint32))
    assert strs.read_field(0)["avg_field_len"] == np.float32(f.avg_field_len)
    one = ob.StringFieldStorage(ctx, data)
    for limit, offset, thr in ((10, 0, None), (100, 0, None), (10, 5, 0.5)):
        p = dict(mode=MODE_FULLTEXT, limit_hint=limit, offset=offset, threshold=thr)
        got = TokenScoreContext(ctx, None, strs).execute_batch_arrays(TokenScoreParams(sharded=True, **p), texts)
        want = TokenScoreContext(ctx, None, one).execute_batch_arrays(TokenScoreParams(**p), texts)
        for a, b in zip(got, want):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (rank, limit, offset, thr)
    one.close()
    strs.close()
    dist.barrier()
    if rank == 0:
        print("SYNC_OK")
    dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
