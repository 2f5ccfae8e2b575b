"""Two processes on the GPU: every rank's ``evaluate(size)`` of the three metrics, with the IoU from
esb_box3d_best_overlap, equals the single-process ``evaluate()`` on the same card over the unpadded samples (the cases
of tests/eval_dist_util.py). Over gloo with both ranks on cuda:0 (records travel as host tensors), and over NCCL with
one GPU per rank when two are visible (device tensors; skipped otherwise)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import eval_dist_util as U

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, backend, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = dict(device_id=dev) if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        q.put((rank, U.on_rank(rank, world, device=dev)))
    finally:
        dist.destroy_process_group()


def _run(backend, world=2):
    want = U.single_process(device='cuda:0')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() * 5 + len(backend)) % 2000
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(60)
    for rank in range(world):
        assert U.first_difference(got[rank], want) is None, (rank, U.first_difference(got[rank], want))
        assert got[rank] == want
    assert want['det']['mAP_0.25'] > 0 and want['ground']['Overall@0.25'] > 0


def test_gloo_two_ranks_on_one_gpu():
    _run('gloo')


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_nccl_two_gpus():
    _run('nccl')
