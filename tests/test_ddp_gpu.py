"""2 GPUs over NCCL: the gradient arena after the bucketed, hook-launched all-reduce of a real detector step (2D side
stream overlap ON, direct-accumulation sparse-conv / BatchNorm gradients) equals the sum of the two ranks' single-rank
gradients (SURVEY §4 (iv); engine.DataParallelReducer). Skipped on a one-GPU box."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import OptimWrapper, broadcast_parameters
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    torch.manual_seed(0)
    cfg = mv_det3d_config('C1')
    model = MODELS.build(cfg).to(dev).train()
    model.overlap_2d_3d = True
    optim = OptimWrapper(model, bucket_bytes=1 << 20)        # many buckets, some mixing 2D and 3D parameters
    broadcast_parameters(optim.arena)
    arena, red = optim.arena, optim.reducer
    batches = [synth_batch(10 + r, 1, n_views=2, H=240, W=320, n_points=2000, device=dev) for r in range(world)]

    # the head normalises its losses by the mean over ranks of the positives per scan (fcaf3d_head.py:1183, dist_utils.py:9):
    # the single-rank passes must use the normaliser of the distributed pass, not their own
    head, store = model.bbox_head, {}
    orig_reduce = head._reduce_mean

    def recording(x):
        store['n_pos'] = orig_reduce(x).clone()
        return store['n_pos']

    def grads(b, reduce):
        head._reduce_mean = recording if reduce else (lambda x: store['n_pos'].clone())
        arena.zero_grad()
        red.reset()
        red.enabled = reduce
        data = model.data_preprocessor(dict(inputs=b['inputs'], data_samples=b['data_samples']), True)
        losses = model(**data, mode='loss')
        sum(losses.values()).backward()
        red.finish()
        torch.cuda.synchronize()
        return arena.grad.clone()

    for m in model.modules():                 # running statistics must not drift between the passes below
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = 0.0
    g_dist = grads(batches[rank], True)
    singles = [grads(batches[r], False) for r in range(world)]
    want = sum(singles)
    scale = float(want.abs().max())
    err = float((g_dist - want).abs().max())
    q.put((rank, err, scale, len(arena.buckets), float(g_dist.abs().sum())))
    dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_nccl_bucketed_gradients_equal_sum_of_single_rank_gradients():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(2)])
    for p in procs:
        p.join(60)
    for rank, err, scale, n_buckets, total in res:
        assert n_buckets > 3 and total > 0
        assert err <= 1e-4 * scale, (rank, err, scale)     # fp32 atomics reorder sums; nothing coarser is allowed
