"""Detection evaluation on the device (SURVEY §8f rank 3): the step right after the hot path.

Mirrors ``indoor_eval`` (embodiedscan/eval/indoor_eval.py:225-310) and its helpers ``eval_map_recall`` (:185-222),
``eval_det_cls`` (:57-182), ``average_precision`` (:7-54, 'area' mode) with the same arguments and the same flat
result dict, but not their shape: the reference walks ``classes x images`` in Python and calls pytorch3d's
``box3d_overlap`` once per (class, image). Here

* the best same-class 9-DoF IoU of EVERY prediction and the ground-truth box that gives it come from ONE launch of
  ``esb_box3d_best_overlap`` over all scans (csrc/iou3d.cu): the ground truth is sorted stably by (scan, label) on the
  device, and each prediction is clipped only against the boxes of its own (scan, label) — the only heavy arithmetic;
* the greedy true-positive marking is a closed form: after a stable descending sort by score, a detection is a true
  positive at threshold t iff its best same-class IoU exceeds t and it is the FIRST such detection for that
  (scan, ground-truth box) — one ``np.unique`` per threshold instead of a Python loop over detections.

The two stages are separate functions: :func:`detection_records` reduces samples to per-detection records (label,
score, best same-class IoU, matched box; the ground-truth labels), :func:`map_recall` turns records in sample order into
AP and AR. That split is what the distributed ``evaluate`` exchanges.

Frozen where the reference is ambiguous: ``np.argsort(-confidence)`` (quicksort) leaves equal scores unordered; the
rule here is a stable sort in input order (scans in order, detections in order).

Distributed evaluation. When ``torch.distributed`` is initialised with more than one rank, ``evaluate(size)`` of the
three metrics computes over the samples of every rank, like the reference's mmengine ``BaseMetric.evaluate`` with
``collect_results``, and every rank returns the same dict. Each rank reduces its own samples first (detection records;
grounding hit counts; occupancy confusion counts), and only those reductions travel: two ``all_gather`` for detection,
one ``all_reduce`` for grounding and for occupancy, whatever the number of scans and classes (device tensors over NCCL,
host tensors over gloo). The global order is the one ``collect_results`` rebuilds, and it assumes mmengine's
``DefaultSampler(shuffle=False)``: rank r's k-th sample is dataset index ``k * W + r``, and indices ``>= size`` are the
sampler's padding duplicates and are dropped. With ``batchwise_anns=True`` (the continuous configs) one ``process`` call
holds the frame prefixes of one scan, so the rule applies to the k-th ``process`` call instead and keeps every prefix
of every real scan in order. This deliberately differs from the reference, which in that mode passes its local
``len(self.results)`` as ``size``, so that mmengine's ``zip`` of the rank parts drops results whenever the ranks hold
different numbers of them. Without ``torch.distributed`` (or with one rank) ``evaluate`` computes over the local results
and ignores ``size``, as before.
"""
from typing import Callable, Dict, List, NamedTuple, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist

from .registry import Registry

METRICS = Registry('metric')


def average_precision(recalls: np.ndarray, precisions: np.ndarray) -> np.float32:
    """Area under the monotone precision envelope (indoor_eval.py:27-39)."""
    mrec = np.concatenate(([0.], recalls, [1.]))
    mpre = np.concatenate(([0.], precisions, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]
    ind = np.where(mrec[1:] != mrec[:-1])[0]
    return np.float32(np.sum((mrec[ind + 1] - mrec[ind]) * mpre[ind + 1]))


def _cuda_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError('indoor_eval computes the 9-DoF IoU in libesb200.so: a CUDA device is required '
                           '(there is no CPU fallback)')
    return torch.device('cuda', torch.cuda.current_device())


def _as_boxes9(x) -> torch.Tensor:
    t = x.tensor if hasattr(x, 'tensor') else torch.as_tensor(np.asarray(x))
    return t.detach().float().reshape(-1, 9).cpu()


def _gt_boxes9(x) -> torch.Tensor:
    if isinstance(x, (list, tuple)):                       # the reference also accepts a list of single boxes
        return torch.cat([_as_boxes9(b) for b in x]) if len(x) else torch.zeros((0, 9))
    return _as_boxes9(x)


def _clamp_thin(pb: torch.Tensor) -> torch.Tensor:
    """indoor_eval.py:118-123: a prediction with a face area below 2e-4 gets every edge clamped to >= 2e-2."""
    pb = pb.clone()
    w, l, h = pb[:, 3], pb[:, 4], pb[:, 5]
    thin = (w * l < 2e-4) | (w * h < 2e-4) | (h * l < 2e-4)
    pb[thin, 3:6] = pb[thin, 3:6].clamp(min=2e-2)
    return pb


def _corners(boxes9: torch.Tensor, dev: torch.device) -> torch.Tensor:
    from .structures import EulerDepthInstance3DBoxes
    return EulerDepthInstance3DBoxes(boxes9.to(dev), box_dim=9, origin=(.5, .5, .5)).corners


def _corners_per_group(boxes9: torch.Tensor, counts: Sequence[int], dev: torch.device) -> torch.Tensor:
    """Corners of consecutive groups of rows (a scan's predictions, a prompt's targets), one container call per group.
    The container's batched rotation (cuBLAS) rounds differently with the batch size, so one call over all scans would
    move IoUs by up to ~4e-5; per group, every IoU keeps the bits of one ``esb_box3d_overlap`` call per scan."""
    return torch.cat([_corners(b, dev) for b in torch.split(boxes9.to(dev), list(counts))] +
                     [torch.zeros((0, 8, 3), device=dev)])


class DetRecords(NamedTuple):
    """Per-detection records of a list of samples, samples in order: sample s owns the next ``n_pred[s]`` detection
    entries and the next ``n_gt[s]`` ground-truth labels. ``best`` is the best IoU against the ground truth of the same
    sample and label (-inf without one), ``arg`` the index of that box within its sample's ground truth (0 without
    one)."""
    n_pred: np.ndarray       # (S,) int64
    pred_label: np.ndarray   # (P,) int64
    score: np.ndarray        # (P,) float64
    best: np.ndarray         # (P,) float32
    arg: np.ndarray          # (P,) int64
    n_gt: np.ndarray         # (S,) int64
    gt_label: np.ndarray     # (G,) int64


def _labels(gt_annos, dt_annos):
    pls = [torch.as_tensor(da['labels_3d']).long().reshape(-1).cpu() for da in dt_annos]
    gls = [torch.as_tensor(np.asarray(ga['gt_labels_3d'])).long().reshape(-1) for ga in gt_annos]
    return pls, gls


def _records(pls, gls, scores, best, arg) -> DetRecords:
    cat = (lambda xs, dt: np.concatenate(xs).astype(dt, copy=False) if xs else np.zeros(0, dt))
    return DetRecords(np.array([p.numel() for p in pls], np.int64), cat([p.numpy() for p in pls], np.int64),
                      cat(scores, np.float64), np.asarray(best, np.float32), np.asarray(arg, np.int64),
                      np.array([g.numel() for g in gls], np.int64), cat([g.numpy() for g in gls], np.int64))


def _scores(da) -> np.ndarray:
    return torch.as_tensor(da['scores_3d']).double().reshape(-1).cpu().numpy()


def _records_from_matrix(gt_annos, dt_annos, iou_fn: Callable) -> DetRecords:
    """Stage (a) through an injected ``iou_fn(pred (m,9), gt (n,9)) -> (m,n)``, one matrix per scan masked to equal
    labels (lets a test substitute a reference IoU)."""
    pls, gls = _labels(gt_annos, dt_annos)
    score, best, arg = [], [], []
    for pl, gl, ga, da in zip(pls, gls, gt_annos, dt_annos):
        m = pl.numel()
        if m == 0:
            continue
        pb = _clamp_thin(_as_boxes9(da['bboxes_3d']))
        gb = _gt_boxes9(ga['gt_bboxes_3d'])
        if gb.shape[0]:
            iou = iou_fn(pb, gb).float().cpu()
            iou = torch.where(pl[:, None] == gl[None, :], iou, torch.full_like(iou, -1.0))
            # strict '>' scan over j (indoor_eval.py:158-163) = first maximum; no same-class box -> -inf
            b, a = iou.max(dim=1)
            has = (pl[:, None] == gl[None, :]).any(1)
            b = torch.where(has, b, torch.full_like(b, float('-inf')))
        else:
            b, a = torch.full((m, ), float('-inf')), torch.zeros(m, dtype=torch.long)
        score.append(_scores(da))
        best.append(b.numpy())
        arg.append(a.numpy())
    cat = (lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt))
    return _records(pls, gls, score, cat(best, np.float32), cat(arg, np.int64))


def same_class_ranges(pscan: torch.Tensor, plabel: torch.Tensor, gscan: torch.Tensor, glabel: torch.Tensor):
    """Ground-truth boxes sorted stably by (scan, label), and for each prediction the range of that order holding the
    boxes of its own (scan, label) -> (tidx, qbeg, qend), the inputs of ``box3d_best_overlap``. Integer tensors on one
    device; the labels are renumbered densely first so that the (scan, label) key cannot overflow."""
    lab, inv = torch.unique(torch.cat([plabel, glabel]), return_inverse=True)
    P = plabel.numel()
    pkey = pscan.long() * lab.numel() + inv[:P]
    gsorted, tidx = torch.sort(gscan.long() * lab.numel() + inv[P:], stable=True)
    return tidx, torch.searchsorted(gsorted, pkey), torch.searchsorted(gsorted, pkey, right=True)


def _records_on_device(gt_annos, dt_annos) -> DetRecords:
    """Stage (a) in one ``esb_box3d_best_overlap`` launch: the ground truth of all samples sorted stably by (sample,
    label) on the device, each prediction's range = the boxes of its own (sample, label); one read-back of the best IoU
    and the matched index of every prediction."""
    from .geometry import box3d_best_overlap
    dev = _cuda_device()
    pls, gls = _labels(gt_annos, dt_annos)
    live = [i for i, pl in enumerate(pls) if pl.numel()]
    n_pred = torch.tensor([pls[i].numel() for i in live], dtype=torch.long)
    n_gt = torch.tensor([gls[i].numel() for i in live], dtype=torch.long)
    P, G = int(n_pred.sum()), int(n_gt.sum())
    best, arg = np.full(P, -np.inf, np.float32), np.zeros(P, np.int64)
    if P and G:
        pb = torch.cat([_clamp_thin(_as_boxes9(dt_annos[i]['bboxes_3d'])) for i in live])
        gb = torch.cat([_gt_boxes9(gt_annos[i]['gt_bboxes_3d']) for i in live])
        assert pb.shape[0] == P and gb.shape[0] == G, 'every box needs one label'
        sample = torch.arange(len(live))
        tidx, qbeg, qend = same_class_ranges(torch.repeat_interleave(sample, n_pred).to(dev),
                                             torch.cat([pls[i] for i in live]).to(dev),
                                             torch.repeat_interleave(sample, n_gt).to(dev),
                                             torch.cat([gls[i] for i in live]).to(dev))
        cq, ct = _corners_per_group(pb, n_pred.tolist(), dev), _corners_per_group(gb, n_gt.tolist(), dev)
        b, a = box3d_best_overlap(cq, ct, tidx, qbeg, qend)
        ba = torch.stack([b.view(torch.int32), a]).cpu()
        best = ba[0].view(torch.float32).numpy()
        a = ba[1].long().numpy()
        goff = np.repeat(np.cumsum(n_gt.numpy()) - n_gt.numpy(), n_pred.numpy())   # first box of each prediction's scan
        arg = np.where(a >= 0, a - goff, 0)
    return _records(pls, gls, [_scores(dt_annos[i]) for i in live], best, arg)


def detection_records(gt_annos: Sequence[dict], dt_annos: Sequence[dict],
                      iou_fn: Optional[Callable] = None) -> DetRecords:
    """Stage (a) of :func:`eval_map_recall`: per-sample records computed from that sample alone. ``iou_fn`` (a test
    hook) replaces the CUDA kernel by an (m,n) IoU matrix per scan."""
    assert len(dt_annos) == len(gt_annos)
    if iou_fn is not None:
        return _records_from_matrix(gt_annos, dt_annos, iou_fn)
    return _records_on_device(gt_annos, dt_annos)


def map_recall(r: DetRecords, metric: Sequence[float]):
    """Stage (b) of :func:`eval_map_recall`: -> (rec, prec, ap) from records in sample order."""
    S = r.n_pred.size
    scan = np.repeat(np.arange(S, dtype=np.int64), r.n_pred)
    label, score, best, arg = r.pred_label, r.score, r.best, r.arg
    gt_labels = np.split(r.gt_label, np.cumsum(r.n_gt)[:-1]) if S else []
    pred_labels = np.split(r.pred_label, np.cumsum(r.n_pred)[:-1]) if S else []
    npos: Dict[int, int] = {}
    for gl in gt_labels:
        for lb, c in zip(*np.unique(gl, return_counts=True)):
            npos[int(lb)] = npos.get(int(lb), 0) + int(c)
    order_of_classes: Dict[int, None] = {}                  # insertion order of the reference's `gt` dict (:254-281)
    for pl, gl in zip(pred_labels, gt_labels):
        for x in pl.tolist() + gl.tolist():
            order_of_classes.setdefault(int(x))
    gt_classes = list(order_of_classes)
    rec = [dict() for _ in metric]
    prec = [dict() for _ in metric]
    ap = [dict() for _ in metric]
    max_gt = max([len(g) for g in gt_labels] + [1])
    for lb in gt_classes:
        sel = np.nonzero(label == lb)[0]
        if sel.size == 0:                                   # class without predictions (indoor_eval.py:217-220)
            for t in range(len(metric)):
                rec[t][lb], prec[t][lb], ap[t][lb] = np.zeros(1), np.zeros(1), np.zeros(1)
            continue
        order = sel[np.argsort(-score[sel], kind='stable')]
        key = scan[order] * max_gt + arg[order]             # (scan, matched ground-truth box)
        n = float(npos.get(lb, 0))
        for t, thr in enumerate(metric):
            hit = best[order] > thr
            tp = np.zeros(order.size)
            first = np.unique(key[hit], return_index=True)[1]
            tp[np.nonzero(hit)[0][first]] = 1.0
            ctp, cfp = np.cumsum(tp), np.cumsum(1.0 - tp)
            with np.errstate(divide='ignore', invalid='ignore'):
                recall = ctp / n
            precision = ctp / np.maximum(ctp + cfp, np.finfo(np.float64).eps)
            rec[t][lb], prec[t][lb] = recall, precision
            ap[t][lb] = np.array([average_precision(recall, precision)], dtype=np.float32)
    return rec, prec, ap


def eval_map_recall(gt_annos, dt_annos, metric: Sequence[float], iou_fn: Optional[Callable] = None):
    """-> (rec, prec, ap): per threshold a dict label -> recall array / precision array / AP, like
    embodiedscan/eval/indoor_eval.py:185-222."""
    return map_recall(detection_records(gt_annos, dt_annos, iou_fn), metric)


def indoor_eval(gt_annos: List[dict], dt_annos: List[dict], metric: Sequence[float], label2cat, logger=None,
                box_mode_3d=None, classes_split=None, iou_fn: Optional[Callable] = None) -> Dict[str, float]:
    """Same call and result keys as the reference's ``indoor_eval``: ``{cat}_AP_{thr}``, ``{cat}_rec_{thr}``,
    ``mAP_{thr}``, ``mAR_{thr}`` (+ ``{split}_mAP_/mAR_{thr}`` when ``classes_split`` is given; the reference only
    prints those). ``gt_annos[i]``: ``gt_bboxes_3d`` (box container or (n,9)), ``gt_labels_3d``; ``dt_annos[i]``:
    ``bboxes_3d``, ``scores_3d``, ``labels_3d``. ``iou_fn(pred (m,9), gt (n,9)) -> (m,n)`` defaults to the CUDA kernel."""
    assert len(dt_annos) == len(gt_annos)
    rec, prec, ap = eval_map_recall(gt_annos, dt_annos, metric, iou_fn)
    return _result_dict(rec, prec, ap, metric, label2cat, classes_split)


def _result_dict(rec, prec, ap, metric, label2cat, classes_split) -> Dict[str, float]:
    for key in list(ap[0].keys()):                          # classes without ground truth: recall = 0/0
        if np.isnan(ap[0][key][0]):
            for d in rec + prec + ap:
                del d[key]
    ret = {}
    for i, thr in enumerate(metric):
        for lb in ap[i]:
            ret[f'{label2cat[lb]}_AP_{thr:.2f}'] = float(ap[i][lb][0])
        ret[f'mAP_{thr:.2f}'] = float(np.mean(list(ap[i].values())))
        rec_list = []
        for lb in rec[i]:
            ret[f'{label2cat[lb]}_rec_{thr:.2f}'] = float(rec[i][lb][-1])
            rec_list.append(rec[i][lb][-1])
        ret[f'mAR_{thr:.2f}'] = float(np.mean(rec_list))
    if classes_split is not None:
        for name, members in zip(('head', 'common', 'tail'), classes_split):
            for i, thr in enumerate(metric):
                aps = [float(ap[i][lb][0]) for lb in members if lb in ap[i]]
                recs = [float(rec[i][lb][-1]) for lb in members if lb in rec[i]]
                if aps:
                    ret[f'{name}_mAP_{thr:.2f}'] = float(np.mean(aps))
                    ret[f'{name}_mAR_{thr:.2f}'] = float(np.mean(recs))
    return ret


# ------------------------------------------------------------------------------------------- distributed evaluate(size)
def _world():
    """(rank, world size) when torch.distributed runs more than one rank, else None."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_rank(), dist.get_world_size()
    return None


def _comm_device() -> torch.device:
    return torch.device('cuda', torch.cuda.current_device()) if dist.get_backend() == 'nccl' else torch.device('cpu')


def _all_gather_int64(x: np.ndarray) -> List[np.ndarray]:
    """Every rank's int64 vector, in rank order: one all_gather of the lengths, one of the vectors padded to the
    longest."""
    dev, world = _comm_device(), dist.get_world_size()
    n = torch.tensor([x.size], dtype=torch.int64, device=dev)
    ns = [torch.empty_like(n) for _ in range(world)]
    dist.all_gather(ns, n)
    ns = [int(v) for v in ns]
    buf = torch.zeros(max(ns + [1]), dtype=torch.int64, device=dev)
    buf[:x.size] = torch.from_numpy(np.ascontiguousarray(x, np.int64)).to(dev)
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf)
    return [p[:k].cpu().numpy() for p, k in zip(parts, ns)]


def _all_reduce_int64(x: np.ndarray) -> np.ndarray:
    t = torch.from_numpy(np.ascontiguousarray(x, np.int64)).to(_comm_device())
    dist.all_reduce(t)
    return t.cpu().numpy()


def _pack_records(r: DetRecords, keys: np.ndarray) -> np.ndarray:
    """Records + per-sample (S,2) order keys -> one int64 vector (floats travel as their bit patterns)."""
    S, P, G = r.n_pred.size, r.pred_label.size, r.gt_label.size
    return np.concatenate([np.array([S, P, G], np.int64), keys.reshape(-1), r.n_pred, r.n_gt, r.pred_label,
                           r.score.view(np.int64), r.best.view(np.int32).astype(np.int64), r.arg, r.gt_label])


def _merge_records(parts: List[np.ndarray]) -> DetRecords:
    """Unpack every rank's records and put the samples in the order of their keys."""
    fields = {k: [] for k in ('keys', 'n_pred', 'n_gt', 'pred_label', 'score', 'best', 'arg', 'gt_label')}
    for buf in parts:
        S, P, G = (int(v) for v in buf[:3])
        o = 3
        for name, n in (('keys', 2 * S), ('n_pred', S), ('n_gt', S), ('pred_label', P), ('score', P), ('best', P),
                        ('arg', P), ('gt_label', G)):
            fields[name].append(buf[o:o + n])
            o += n
    f = {k: np.concatenate(v) for k, v in fields.items()}
    keys = f['keys'].reshape(-1, 2)
    order = np.lexsort((keys[:, 1], keys[:, 0]))

    def gather(counts):                     # element indices of the samples' segments, samples in `order`
        off = np.cumsum(counts) - counts
        return np.concatenate([np.arange(off[i], off[i] + counts[i]) for i in order] + [np.zeros(0, np.int64)])

    p, g = gather(f['n_pred']), gather(f['n_gt'])
    return DetRecords(f['n_pred'][order], f['pred_label'][p], f['score'][p].view(np.float64),
                      f['best'][p].astype(np.int32).view(np.float32), f['arg'][p], f['n_gt'][order],
                      f['gt_label'][g])


class _RankedResults:
    """What the three metrics share for ``evaluate(size)`` under torch.distributed: the ``process`` call each result
    came from, and which local results are real samples and where they go in dataset order (module docstring)."""
    batchwise_anns = False

    def _reset(self):
        if not hasattr(self, 'results'):
            self.results, self._call_of = [], []
        self.results.clear()
        self._call_of.clear()
        self._calls = 0

    def _mark_call(self, n_before: int) -> None:
        """Called at the end of ``process``: the results appended since ``n_before`` belong to one call."""
        self._call_of += [self._calls] * (len(self.results) - n_before)
        self._calls += 1

    def _local_order(self, rank: int, world: int, size: Optional[int]):
        """-> (indices of the local results that are not padding, their (S,2) int64 keys in global order)."""
        keep, keys, first = [], [], {}
        for k in range(len(self.results)):
            if self.batchwise_anns:                       # k-th process call = scan c*W + r; its prefixes in order
                c = self._call_of[k]
                key = (c * world + rank, k - first.setdefault(c, k))
            else:                                         # k-th sample = dataset index k*W + r
                key = (k * world + rank, 0)
            if size is None or key[0] < size:
                keep.append(k)
                keys.append(key)
        return keep, np.array(keys, np.int64).reshape(-1, 2)

    def _with_prefix(self, out: Dict[str, float]) -> Dict[str, float]:
        return {'/'.join((self.prefix, k)): v for k, v in out.items()} if self.prefix else out


@METRICS.register_module()
class IndoorDetMetric(_RankedResults):
    """``embodiedscan/eval/metrics/det_metric.py`` IndoorDetMetric: collects ``(eval_ann_info, pred_instances_3d)``
    pairs from ``process`` and evaluates them with :func:`indoor_eval`, over every rank under torch.distributed (module
    docstring). ``iou_fn`` is :func:`indoor_eval`'s test hook."""

    def __init__(self, iou_thr=(0.25, 0.5), collect_device='cpu', prefix=None, batchwise_anns=False,
                 iou_fn: Optional[Callable] = None, **kwargs):
        self.iou_thr = [iou_thr] if isinstance(iou_thr, float) else list(iou_thr)
        self.prefix, self.dataset_meta = prefix, {}
        self.batchwise_anns, self.iou_fn = batchwise_anns, iou_fn
        self._reset()

    def process(self, data_batch, data_samples) -> None:
        n0 = len(self.results)
        for ds in data_samples:
            get = ds.get if hasattr(ds, 'get') else ds.__getitem__
            pred = get('pred_instances_3d')
            ann = get('eval_ann_info')
            self.results.append((ann, dict(bboxes_3d=pred['bboxes_3d'] if isinstance(pred, dict) else pred.bboxes_3d,
                                           scores_3d=pred['scores_3d'] if isinstance(pred, dict) else pred.scores_3d,
                                           labels_3d=pred['labels_3d'] if isinstance(pred, dict) else pred.labels_3d)))
        self._mark_call(n0)

    def compute_metrics(self, results=None) -> Dict[str, float]:
        results = self.results if results is None else results
        anns, preds = zip(*results) if results else ((), ())
        out = indoor_eval(list(anns), list(preds), self.iou_thr, self.dataset_meta['classes'],
                          classes_split=self.dataset_meta.get('classes_split'), iou_fn=self.iou_fn)
        return self._with_prefix(out)

    def evaluate(self, size=None) -> Dict[str, float]:
        ws = _world()
        if ws is None:
            out = self.compute_metrics()
        else:
            keep, keys = self._local_order(*ws, size)
            anns = [self.results[k][0] for k in keep]
            preds = [self.results[k][1] for k in keep]
            local = detection_records(anns, preds, self.iou_fn)
            merged = _merge_records(_all_gather_int64(_pack_records(local, keys)))
            rec, prec, ap = map_recall(merged, self.iou_thr)
            out = self._with_prefix(_result_dict(rec, prec, ap, self.iou_thr, self.dataset_meta['classes'],
                                                 self.dataset_meta.get('classes_split')))
        self._reset()
        return out


@METRICS.register_module()
class GroundingMetric(_RankedResults):
    """``embodiedscan/eval/metrics/grounding_metric.py``: a prompt counts as found at threshold t when one of its 10
    highest-scoring boxes overlaps a target box with 9-DoF IoU > t; accuracy overall and per Easy/Hard,
    View-Dep/View-Indep, Unique/Multi split. The candidates of all prompts are matched against their prompts' targets in
    one ``esb_box3d_best_overlap`` launch (a prompt is found at t iff a candidate's best IoU exceeds t).
    Frozen: the top-10 come from a STABLE descending sort (torch's default argsort leaves ties unordered).
    Under torch.distributed each rank counts its prompts and the counts are summed (module docstring)."""

    TYPES = ('Easy', 'Hard', 'View-Dep', 'View-Indep', 'Unique', 'Multi', 'Overall')

    def __init__(self, iou_thr=(0.25, 0.5), collect_device='cpu', prefix=None, format_only=False, result_dir='',
                 iou_fn: Optional[Callable] = None, **kw):
        self.iou_thr = [iou_thr] if isinstance(iou_thr, float) else list(iou_thr)
        self.prefix, self.iou_fn = prefix, iou_fn
        self._reset()

    def process(self, data_batch, data_samples) -> None:
        n0 = len(self.results)
        for ds in data_samples:
            get = ds.get if hasattr(ds, 'get') else ds.__getitem__
            pred = get('pred_instances_3d')
            pred = dict(pred.items()) if hasattr(pred, 'items') else {k: getattr(pred, k) for k in pred.keys()}
            self.results.append((get('eval_ann_info'), pred))
        self._mark_call(n0)

    def _found(self, gt_annos, det_annos, iou_fn: Optional[Callable]) -> torch.Tensor:
        """(prompts, thresholds) bool: one of the prompt's 10 best-scoring boxes has IoU > t with one of its targets."""
        thr = torch.tensor(self.iou_thr, dtype=torch.float32)
        cands = [_as_boxes9(det['bboxes_3d'])[torch.sort(torch.as_tensor(det['target_scores_3d']).reshape(-1),
                                                         descending=True, stable=True).indices[:10].cpu()]
                 for det in det_annos]
        tgts = [_gt_boxes9(ann['gt_bboxes_3d']) for ann in gt_annos]
        if iou_fn is not None:
            return torch.stack([(iou_fn(c, t).float().cpu().reshape(-1, 1) > thr).any(0) for c, t in zip(cands, tgts)]
                               ) if cands else torch.zeros((0, thr.numel()), dtype=torch.bool)
        from .geometry import box3d_best_overlap
        dev = _cuda_device()
        nc = torch.tensor([c.shape[0] for c in cands], dtype=torch.long)
        nt = torch.tensor([t.shape[0] for t in tgts], dtype=torch.long)
        if int(nc.sum()) == 0 or int(nt.sum()) == 0:
            return torch.zeros((len(cands), thr.numel()), dtype=torch.bool)
        toff = torch.cumsum(nt, 0) - nt
        qbeg = torch.repeat_interleave(toff, nc)
        qend = qbeg + torch.repeat_interleave(nt, nc)
        cq = _corners_per_group(torch.cat(cands), nc.tolist(), dev)
        ct = _corners_per_group(torch.cat(tgts), nt.tolist(), dev)
        best = box3d_best_overlap(cq, ct, torch.arange(ct.shape[0], device=dev), qbeg.to(dev), qend.to(dev))[0].cpu()
        prompt = torch.repeat_interleave(torch.arange(len(cands)), nc)
        found = torch.zeros((len(cands), thr.numel()), dtype=torch.long)
        found.index_add_(0, prompt, (best[:, None] > thr).long())
        return found > 0

    def _counts(self, gt_annos, found: torch.Tensor) -> np.ndarray:
        """(2, thresholds, TYPES) int64: prompts per (threshold, tag), and how many of them were found."""
        cnt = np.zeros((2, len(self.iou_thr), len(self.TYPES)), np.int64)
        for ann, f in zip(gt_annos, found.tolist()):
            tags = ('View-Dep' if ann['is_view_dep'] else 'View-Indep', 'Hard' if ann['is_hard'] else 'Easy',
                    'Unique' if ann['is_unique'] else 'Multi', 'Overall')
            for tag in tags:
                o = self.TYPES.index(tag)
                cnt[0, :, o] += 1
                cnt[1, :, o] += np.asarray(f, np.int64)
        return cnt

    def _accuracy(self, cnt: np.ndarray) -> Dict[str, float]:
        out = {}
        for i, t in enumerate(self.iou_thr):
            for o, name in enumerate(self.TYPES):
                total = 1e-14                     # the reference's float counter, one prompt at a time
                for _ in range(int(cnt[0, i, o])):
                    total += 1
                out[f'{name}@{t}'] = int(cnt[1, i, o]) / max(total, 1)
        return out

    def ground_eval(self, gt_annos, det_annos, iou_fn: Optional[Callable] = None) -> Dict[str, float]:
        assert len(det_annos) == len(gt_annos)
        return self._accuracy(self._counts(gt_annos, self._found(gt_annos, det_annos, iou_fn or self.iou_fn)))

    def compute_metrics(self, results=None) -> Dict[str, float]:
        results = self.results if results is None else results
        anns, preds = zip(*results) if results else ((), ())
        return self._with_prefix(self.ground_eval(list(anns), list(preds)))

    def evaluate(self, size=None):
        ws = _world()
        if ws is None:
            out = self.compute_metrics()
        else:
            keep = self._local_order(*ws, size)[0]
            anns = [self.results[k][0] for k in keep]
            dets = [self.results[k][1] for k in keep]
            cnt = _all_reduce_int64(self._counts(anns, self._found(anns, dets, self.iou_fn)))
            out = self._with_prefix(self._accuracy(cnt))
        self._reset()
        return out


@METRICS.register_module()
class OccupancyMetric(_RankedResults):
    """``embodiedscan/eval/metrics/occupancy_metric.py``: per-class IoU of the arg-max occupancy (class 0 = geometry:
    occupied vs empty), voxels with ground truth 255 (invisible) ignored. The per-scan counts are three ``bincount``s
    on whatever device holds the prediction instead of ``num_class`` masked passes; under torch.distributed the integer
    counts of every rank are summed (module docstring)."""

    def __init__(self, collect_device='cpu', prefix=None, batchwise_anns=False, **kw):
        self.prefix, self.dataset_meta, self.batchwise_anns = prefix, {}, batchwise_anns
        self._reset()

    def process(self, data_batch, data_samples) -> None:
        n0 = len(self.results)
        for ds in data_samples:
            get = ds.get if hasattr(ds, 'get') else ds.__getitem__
            pred = get('pred_occupancy')
            gt4 = get('gt_occupancy').long().to(pred.device)
            gt = torch.zeros_like(pred)
            gt[gt4[:, 0], gt4[:, 1], gt4[:, 2]] = gt4[:, 3].to(pred.dtype)
            if 'gt_occupancy_masks' in ds:
                gt[~get('gt_occupancy_masks').to(pred.device)] = 255
            self.results.append((gt, pred))
        self._mark_call(n0)

    def _counts(self, results) -> np.ndarray:
        """(n_class + 1, 3) int64 (true positives, ground truth, prediction) summed over the samples."""
        n = len(self.dataset_meta['classes']) + 1
        score = torch.zeros((n, 3), dtype=torch.int64)
        for gt, pred in results:
            keep = gt != 255
            g, p = gt[keep].long().clamp(max=n - 1), pred[keep].long().clamp(max=n - 1)
            tp = torch.bincount(g[g == p], minlength=n)
            cg, cp = torch.bincount(g, minlength=n), torch.bincount(p, minlength=n)
            cnt = torch.stack([tp, cg, cp], 1)
            cnt[0] = torch.stack([((g != 0) & (p != 0)).sum(), (g != 0).sum(), (p != 0).sum()])
            score += cnt.cpu()
        return score.numpy()

    def _ious(self, score: np.ndarray) -> Dict[str, float]:
        classes = self.dataset_meta['classes']
        ret = {}
        for i in range(len(classes) + 1):
            tp, a, b = (float(x) for x in score[i])
            union = a + b - tp
            if union == 0:                       # the reference skips classes whose IoU is 0/0
                continue
            ret['empty' if i == 0 else classes[i - 1]] = tp / union
        return self._with_prefix(ret)

    def compute_metrics(self, results=None) -> Dict[str, float]:
        return self._ious(self._counts(self.results if results is None else results))

    def evaluate(self, size=None):
        ws = _world()
        if ws is None:
            out = self.compute_metrics()
        else:
            keep = self._local_order(*ws, size)[0]
            out = self._ious(_all_reduce_int64(self._counts([self.results[k] for k in keep])))
        self._reset()
        return out
