"""CPU, W = 2 and W = 3 over gloo: ``evaluate(size)`` of IndoorDetMetric, GroundingMetric and OccupancyMetric on every
rank equals the single-process ``evaluate()`` over the unpadded samples in dataset order, with the golden fixtures split
as mmengine's DefaultSampler splits them (padding duplicates, a rank left with padding only, several samples per
``process`` call, ``batchwise_anns`` scans with unequal prefix counts per rank, ``prefix=``). The IoU is the oracle's,
injected as in tests/test_golden_cpu.py; the single-process results are pinned to the reference's goldens here too."""
import json
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import eval_dist_util as U


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        q.put((rank, U.on_rank(rank, world, iou_fn=U.oracle_iou)))
    finally:
        dist.destroy_process_group()


def _spawn(world):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() * 7 + world) % 2000
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(60)
    return res


def test_single_process_results_match_the_reference_goldens():
    g = np.load(os.path.join(U.HERE, 'golden', 'metrics.npz'))
    want_det = json.loads(str(np.load(os.path.join(U.HERE, 'golden', 'eval.npz'))['result_json']))
    got = U.single_process(iou_fn=U.oracle_iou)
    for name, want, tol in (('det', want_det, 1e-6), ('ground', json.loads(str(g['grounding_json'])), 1e-12),
                            ('occ', json.loads(str(g['occupancy_json'])), 1e-12)):
        assert set(want) <= set(got[name]), name
        for k in want:
            assert abs(got[name][k] - want[k]) <= tol, (name, k, got[name][k], want[k])
    assert {'head_mAP_0.25', 'common_mAR_0.50', 'tail_mAP_0.50'} <= set(got['det'])       # classes_split rows


@pytest.mark.parametrize('world', [2, 3])
def test_every_rank_returns_the_single_process_result(world):
    want = U.single_process(iou_fn=U.oracle_iou)
    got = _spawn(world)
    assert sorted(got) == list(range(world))
    for rank in range(world):
        assert U.first_difference(got[rank], want) is None, (rank, U.first_difference(got[rank], want))
        assert got[rank] == want
    assert set(want['det_batch2_prefix']) == {'val/' + k for k in want['det']}
    assert all(k.startswith('occ/') for k in want['occ_batchwise_prefix'])


def test_shard_is_default_sampler():
    assert [U.shard(4, 3, r) for r in range(3)] == [[0, 3], [1, 0], [2, 1]]
    assert [U.shard(2, 3, r) for r in range(3)] == [[0], [1], [0]]
    assert [U.shard(1, 3, r) for r in range(3)] == [[0], [0], [0]]


def test_same_class_ranges_hold_exactly_the_same_scan_and_label_boxes():
    """The ranges esb_box3d_best_overlap walks, built on the host here: each prediction's range lists the ground truth
    of its own (scan, label), in ascending box order (a stable sort)."""
    import torch
    from embodiedscan_b200.evaluation import same_class_ranges
    g = torch.Generator().manual_seed(3)
    pscan, gscan = torch.randint(0, 9, (500, ), generator=g), torch.randint(0, 9, (120, ), generator=g)
    pl, gl = torch.randint(0, 284, (500, ), generator=g) * 1000, torch.randint(0, 284, (120, ), generator=g) * 1000
    src = torch.randint(0, 120, (167, ), generator=g)
    pl[::3], pscan[::3] = gl[src], gscan[src]
    tidx, qbeg, qend = same_class_ranges(pscan, pl, gscan, gl)
    mask = (pscan[:, None] == gscan[None]) & (pl[:, None] == gl[None])
    assert int(mask.sum()) > 100
    for i in range(500):
        assert torch.equal(tidx[qbeg[i]:qend[i]], torch.nonzero(mask[i]).flatten()), i
