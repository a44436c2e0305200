"""Evaluation of trained samplers: the numbers the reference reports, restated on device tensors over this package's kernels.

    registration    registration/main.py:364-414 eval_1, :416-483 test_1        RegistrationStep.eval_1 / .test_1 (registration.py; the
                                                                                 precision curve and the mode handling are here)
    classification  classification/evaluate_samplenet.py:156-277                ClassificationEvaluator
                    classification/evaluate_classifier.py:128-222,
                    train_classifier.py:245-301 eval_one_epoch                  ClassifierEvaluator (the classifier alone, rotation votes)
                    classification/infer_samplenet_progressive.py:94-255,
                    classification/evaluate_from_files.py:109-189               ProgressiveClassificationEvaluator
    retrieval       classification/models/pointnet_cls.py:111 (the descriptor;
                    the reference has no retrieval evaluator)                   RetrievalEvaluator, ProgressiveClassificationEvaluator.retrieval
    reconstruction  reconstruction/sampler/evaluate_samplenet(_progressive).py,
                    src/samplenet_pointnet_ae.py:459-492 (get_sample, get_samples),
                    src/sampler_progressive_autoencoder.py:145-177,
                    autoencoder/evaluate_ae.py (the reference loss)             ReconstructionEvaluator

Datasets, h5 / ply files, checkpoints and command lines stay the caller's: every evaluator takes device tensors.  Every loop runs under
torch.no_grad() with the sampler and the task network in eval mode (their modes are restored afterwards), takes a plain task module or
its frozen CUDA wrapper, takes FPSSampler / RandomSampler in place of a learned sampler (they return one tensor, not a pair), and reads
its results back to the host once per call: metrics accumulate on the device.
"""
import contextlib

import numpy as np
import torch

from . import ops, sputils, tasknets, tf_ops

PREFIX_CHUNK = ops.FROZEN_MAX_PREFIX      # sizes per prefixes() call of a wrapper without ONE_PASS_PREFIXES (the encoder's num_prefix limit)


@contextlib.contextmanager
def eval_mode(*modules):
    """Put the modules (None entries are skipped) in eval mode under torch.no_grad(), and give every submodule its own `training` flag
    back afterwards (main.py:368-372, :409-412 does so for the task network and the sampler)."""
    saved = [(m, m.training) for mod in modules if mod is not None for m in mod.modules()]
    try:
        for mod in modules:
            if mod is not None:
                mod.eval()
        with torch.no_grad():
            yield
    finally:
        for m, flag in saved:
            m.training = flag


def _chunks(n, size):
    if size < 1:
        raise ValueError("batch_size must be positive, got %r" % (size,))
    return [(s, min(s + size, n)) for s in range(0, n, size)]


def _sampler_output(out):
    """(simplified, sampled) of a learned sampler's pair, or the one tensor of a baseline sampler as both."""
    return (out[0], out[1]) if isinstance(out, (tuple, list)) else (out, out)


# ----------------------------------------------------------------------------------------------------- metric restatements
def precision_curve(rotation_errors, thresholds=None):
    """main.py:461-477: x = np.arange(0, 180, 0.5) degrees, y[i] = fraction of records with rotation error <= x[i], auc = sum(y) / len(x).
    Returns (x, y, auc)."""
    err = np.asarray(rotation_errors, dtype=np.float64).reshape(-1)
    x = np.arange(0.0, 180.0, 0.5) if thresholds is None else np.asarray(thresholds, dtype=np.float64)
    y = (err[None, :] <= x[:, None]).sum(axis=1) / float(max(err.size, 1))
    return x, y, float(np.sum(y) / len(x))


def classification_counts(logits, labels, num_classes=None):
    """evaluate_samplenet.py:241-258 on tensors of any device: (predictions (n,), seen per class (C,), correct per class (C,)), the two
    counts in float64.  No host synchronisation (index_add_, not bincount)."""
    num_classes = int(logits.shape[1] if num_classes is None else num_classes)
    pred = torch.argmax(logits, dim=1)
    labels = labels.to(pred.device).long().reshape(-1)
    seen = torch.zeros(num_classes, dtype=torch.float64, device=pred.device).index_add_(0, labels, torch.ones_like(labels, dtype=torch.float64))
    correct = torch.zeros(num_classes, dtype=torch.float64, device=pred.device).index_add_(0, labels, (pred == labels).to(torch.float64))
    return pred, seen, correct


def class_accuracies(seen, correct):
    """evaluate_samplenet.py:261-275: (accuracy, per-class accuracy, their mean).  As there, a class without a record divides by zero: its
    entry and the mean are NaN."""
    seen, correct = np.asarray(seen, dtype=np.float64), np.asarray(correct, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        per_class = correct / seen
    return float(correct.sum() / seen.sum()), per_class, float(np.mean(per_class))


def nre(ae_loss_per_pc, ae_loss_per_pc_ref):
    """evaluate_samplenet.py:149-152: the normalised reconstruction error per cloud, the sampled cloud's AE loss over the complete cloud's."""
    if isinstance(ae_loss_per_pc, torch.Tensor):
        return ae_loss_per_pc / ae_loss_per_pc_ref
    return np.divide(ae_loss_per_pc, ae_loss_per_pc_ref)


def _num_unique(idx):
    """np.size(np.unique(idx[i])) per row (evaluate_samplenet.py:227-228), on the device."""
    srt = torch.sort(idx.long(), dim=1)[0]
    return 1 + (srt[:, 1:] != srt[:, :-1]).sum(dim=1)


# ----------------------------------------------------------------------------------------------------- classification
class ClassificationEvaluator:
    """classification/evaluate_samplenet.py:156-277.  `sampler`: a ClassificationSampleNet (or any module returning (simplified,
    projected) on (B, N, 3) clouds) or a baseline sampler with "bnc" shapes; `classifier`: PointNetCls / PointNetClsTransforms or a frozen
    wrapper.  The classifier sees the matched sample (nearest input point of every generated point, order-preserving unique, FPS
    completion to num_out_points) when match_output is true and the simplified points otherwise (:218-225).

    Deviation: the reference drops the clouds after the last whole batch (:179); every cloud is evaluated here."""

    def __init__(self, sampler, classifier, num_out_points, match_output=True):
        self.sampler, self.classifier, self.num_out_points, self.match_output = sampler, classifier, int(num_out_points), bool(match_output)

    def clouds(self, pc):
        """The four clouds infer_samplenet_progressive.py:183-212 saves, and the nearest-neighbour indices, of one batch (eval mode is the
        caller's): {"simplified", "soft_projected", "hard_projected", "sampled", "idx"}.  A sampler without the TF SoftProjection (a
        baseline) has no projection: its output stands for the first three."""
        pc = pc.contiguous()
        simplified, _ = _sampler_output(self.sampler(pc))
        simplified = simplified.contiguous()
        _, idx, _, _ = ops.nn_distance_forward(simplified, pc)
        project = getattr(self.sampler, "project", None)
        if isinstance(project, tf_ops.SoftProjection):
            soft, hard = project(pc, simplified, hard=False)[0], project(pc, simplified, hard=True)[0]
        else:
            soft = hard = simplified
        sampled = sputils.nn_matching_cuda(pc, idx, self.num_out_points)
        return {"simplified": simplified, "soft_projected": soft, "hard_projected": hard, "sampled": sampled, "idx": idx}

    def evaluate(self, point_clouds, labels, batch_size=32, num_classes=None):
        """point_clouds (n, N, 3) and labels (n,) on the device -> {"accuracy", "class_accuracy" (C,), "avg_class_accuracy", "mean_loss",
        "mean_unique_idx", "predictions" (n,) numpy, and the four clouds as device tensors}.  One host read-back."""
        labels = labels.to(point_clouds.device).long().reshape(-1)
        kept = {k: [] for k in ("simplified", "soft_projected", "hard_projected", "sampled")}
        logits, loss_sum, unique_sum = [], 0.0, 0.0
        with eval_mode(self.sampler, self.classifier):
            for s, e in _chunks(point_clouds.shape[0], batch_size):
                c = self.clouds(point_clouds[s:e])
                for k in kept:
                    kept[k].append(c[k])
                pred, end_points = self.classifier(c["sampled"] if self.match_output else c["simplified"])
                loss_sum = loss_sum + self.classifier.get_loss(pred, labels[s:e], end_points).double() * (e - s)      # :244
                unique_sum = unique_sum + _num_unique(c["idx"]).sum().double()
                logits.append(pred)
            logits = torch.cat(logits)
            pred, seen, correct = classification_counts(logits, labels, num_classes)
            n = point_clouds.shape[0]
            packed = torch.cat([torch.stack([loss_sum / n, unique_sum / n]), seen, correct, pred.double()]).cpu().numpy()
        c = seen.numel()
        accuracy, per_class, avg = class_accuracies(packed[2:2 + c], packed[2 + c:2 + 2 * c])
        out = {"accuracy": accuracy, "class_accuracy": per_class, "avg_class_accuracy": avg, "mean_loss": float(packed[0]),
               "mean_unique_idx": float(packed[1]), "predictions": packed[2 + 2 * c:].astype(np.int64)}
        out.update({k: torch.cat(v) for k, v in kept.items()})
        return out


class ClassifierEvaluator:
    """classification/evaluate_classifier.py:128-222 on the classifier alone: every batch is classified num_votes times, vote v rotated about
    the up axis by v / V * 2 pi (all V copies from one ops.rotate_by_angles launch, classified in one call: the frozen wrappers chunk at 64
    clouds themselves); the prediction is the argmax of the logits summed over the votes in float64, in vote order, and the batch's loss is
    sum_v loss_v * b / V.  With num_votes=1 this is also eval_one_epoch (train_classifier.py:245-301), and the clouds go in unrotated (a
    rotation by 0 is the identity bit for bit).  `classifier`: PointNetCls / PointNetClsTransforms or a frozen wrapper.

    get_loss runs once per vote on that vote's rows of the logits and end points: PointNetClsTransforms.get_loss sums its transform
    regulariser over the batch instead of averaging it, so one call on all V * b rows would count the regulariser V times.

    Deviation: the reference drops the clouds after the last whole batch (:148); every cloud is evaluated here."""

    def __init__(self, classifier, num_votes=1):
        if isinstance(num_votes, bool) or int(num_votes) != num_votes or num_votes < 1:
            raise ValueError("num_votes must be a positive integer, got %r" % (num_votes,))
        self.classifier, self.num_votes = classifier, int(num_votes)

    def evaluate(self, point_clouds, labels, batch_size=32, num_classes=None):
        """point_clouds (n, N, 3) and labels (n,) on the device -> {"accuracy", "class_accuracy" (C,), "avg_class_accuracy", "mean_loss",
        "predictions" (n,) numpy}.  One host read-back."""
        V = self.num_votes
        angles = [v / float(V) * np.pi * 2 for v in range(V)]
        labels = labels.to(point_clouds.device).long().reshape(-1)
        logits, loss_sum = [], 0.0
        with eval_mode(self.classifier):
            for s, e in _chunks(point_clouds.shape[0], batch_size):
                b, pc = e - s, point_clouds[s:e].contiguous()
                x = pc if V == 1 else ops.rotate_by_angles(pc, angles).flatten(0, 1)
                pred, end_points = self.classifier(x)
                summed, batch_loss = pred[:b].double(), 0.0
                for v in range(V):
                    rows = slice(v * b, (v + 1) * b)
                    if v:
                        summed = summed + pred[rows].double()
                    ep = {k: (t[rows] if isinstance(t, torch.Tensor) else t) for k, t in end_points.items()}
                    batch_loss = batch_loss + self.classifier.get_loss(pred[rows], labels[s:e], ep).double() * b / V
                loss_sum = loss_sum + batch_loss
                logits.append(summed)
            pred, seen, correct = classification_counts(torch.cat(logits), labels, num_classes)
            n = point_clouds.shape[0]
            packed = torch.cat([(loss_sum / n).reshape(1), seen, correct, pred.double()]).cpu().numpy()
        c = seen.numel()
        accuracy, per_class, avg = class_accuracies(packed[1:1 + c], packed[1 + c:1 + 2 * c])
        return {"accuracy": accuracy, "class_accuracy": per_class, "avg_class_accuracy": avg, "mean_loss": float(packed[0]),
                "predictions": packed[1 + 2 * c:].astype(np.int64)}


class ProgressiveClassificationEvaluator:
    """The progressive sampler's curve: infer_samplenet_progressive.py:94-255 orders every cloud once, evaluate_from_files.py:109-189
    classifies the first s points of that order for every sample size s."""

    def __init__(self, sampler, classifier):
        self.sampler, self.classifier = sampler, classifier

    def order(self, point_clouds, batch_size=32):
        """infer_samplenet_progressive.py:207-212 with NUM_OUT_POINTS = N: one generator pass, the nearest input point of every generated
        point, order-preserving unique, farthest point completion to all N points.  (n, N, 3) -> (n, N, 3), every cloud reordered."""
        out = []
        with eval_mode(self.sampler):
            for s, e in _chunks(point_clouds.shape[0], batch_size):
                pc = point_clouds[s:e].contiguous()
                simplified, _ = _sampler_output(self.sampler(pc))
                _, idx, _, _ = ops.nn_distance_forward(simplified.contiguous(), pc)
                out.append(sputils.nn_matching_cuda(pc, idx, pc.shape[1]))
        return torch.cat(out)

    def _per_size(self, ordered, sizes, end_point=None):
        """(len(sizes), B, ...) of ordered[:, :s]: the logits, or the end point of that name.  A classifier whose prefixes() runs any number
        of sizes in one pass (FrozenPointNetCls: ONE_PASS_PREFIXES) takes them all in one call, one with a 16-size prefixes()
        (FrozenPointNetClsTransforms, whose points depend on the prefix) 16 sizes per call, and a plain module one size per call."""
        sizes = [int(s) for s in sizes]
        if hasattr(self.classifier, "prefixes"):
            asc, parts = sorted(set(sizes)), []
            step = len(asc) if getattr(self.classifier, "ONE_PASS_PREFIXES", False) else PREFIX_CHUNK
            for i in range(0, len(asc), step):
                if end_point is None:
                    parts.append(self.classifier.prefixes(ordered, asc[i:i + step]))
                else:
                    parts.append(torch.stack([ep[end_point] for ep in self.classifier.prefixes(ordered, asc[i:i + step], return_end_points=True)[1]]))
            rows = torch.cat(parts)
            return rows if asc == sizes else rows[[asc.index(s) for s in sizes]]
        outs = [self.classifier(ordered[:, :s].contiguous()) for s in sizes]
        return torch.stack([o[0] if end_point is None else o[1][end_point] for o in outs])

    def logits(self, ordered, sizes):
        """(len(sizes), B, classes) logits of ordered[:, :s]."""
        return self._per_size(ordered, sizes)

    def _prepare(self, point_clouds, labels, sizes, batch_size, ordered):
        sizes = [int(s) for s in sizes]
        if not sizes or min(sizes) < 1 or max(sizes) > point_clouds.shape[1]:
            raise ValueError("sizes must lie in [1, %d]" % point_clouds.shape[1])
        labels = labels.to(point_clouds.device).long().reshape(-1)
        return sizes, labels, self.order(point_clouds, batch_size) if ordered is None else ordered

    def evaluate(self, point_clouds, labels, sizes, batch_size=32, ordered=None):
        """-> {"sizes", "accuracy" (len(sizes),) numpy, "ordered" (n, N, 3) device}: evaluate_from_files.py:158-171 for every size.
        sizes=range(1, N + 1) is the reference's dense evaluation.  One host read-back."""
        sizes, labels, ordered = self._prepare(point_clouds, labels, sizes, batch_size, ordered)
        correct = torch.zeros(len(sizes), dtype=torch.float64, device=point_clouds.device)
        with eval_mode(self.classifier):
            for s, e in _chunks(ordered.shape[0], batch_size):
                pred = torch.argmax(self.logits(ordered[s:e].contiguous(), sizes), dim=2)
                correct += (pred == labels[s:e][None, :]).sum(dim=1)
            accuracy = (correct / ordered.shape[0]).cpu().numpy()
        return {"sizes": sizes, "accuracy": accuracy, "ordered": ordered}

    def retrieval(self, point_clouds, labels, sizes, batch_size=32, ordered=None, recall_levels=11):
        """Leave-one-out retrieval among the descriptors (end_points["retrieval_vectors"]) of ordered[:, :s] for every size s, from the same
        order() as evaluate() and the prefixes() passes of _per_size: {"sizes", "map" (len(sizes),), "precision" (len(sizes), recall_levels)}
        as numpy, each the mean over the queries with a relevant result (see RetrievalEvaluator).  One retrieval_metrics launch per size;
        one host read-back."""
        sizes, labels, ordered = self._prepare(point_clouds, labels, sizes, batch_size, ordered)
        with eval_mode(self.classifier):
            desc = torch.cat([self._per_size(ordered[s:e].contiguous(), sizes, "retrieval_vectors") for s, e in _chunks(ordered.shape[0], batch_size)],
                             dim=1)
            means = [_retrieval_means(ops.retrieval_metrics(desc[p].contiguous(), labels, recall_levels=recall_levels))[0] for p in range(len(sizes))]
            packed = torch.stack(means).cpu().numpy()
        return {"sizes": sizes, "map": packed[:, 0], "precision": packed[:, 1:]}


# ----------------------------------------------------------------------------------------------------- retrieval
def _retrieval_means(metrics):
    """(packed [map, mean precision curve (L,)] float64, queries with a relevant result) over those queries, on the device."""
    valid = metrics["num_relevant"] > 0
    count = valid.sum().double()
    ap = torch.where(valid, metrics["ap"], torch.zeros_like(metrics["ap"])).sum() / count
    curve = torch.where(valid[:, None], metrics["precision"], torch.zeros_like(metrics["precision"])).sum(dim=0) / count
    return torch.cat([ap.reshape(1), curve]), count


class RetrievalEvaluator:
    """Shape retrieval with a classifier's descriptors (end_points["retrieval_vectors"], fc3's input; classification/models/pointnet_cls.py:111),
    scored by ops.retrieval_metrics: every query ranks the database by squared L2 distance, ties by index, and the metrics are average
    precision and the interpolated precision curve.  The reference ships no retrieval evaluator; the paper's exact query / database split
    stays the caller's.  `sampler`: as ClassificationEvaluator's (its clouds() samples and matches), or None to evaluate the clouds as given
    (the complete-cloud baseline); `classifier`: PointNetCls / PointNetClsTransforms or a frozen wrapper."""

    def __init__(self, sampler, classifier, num_out_points, match_output=True):
        self.sampler, self.classifier, self.num_out_points, self.match_output = sampler, classifier, int(num_out_points), bool(match_output)
        self._clouds = ClassificationEvaluator(sampler, classifier, num_out_points, match_output)

    def descriptors(self, point_clouds, batch_size=32, sampled=True):
        """(n, 256) descriptors of the sampled clouds (the matched sample with match_output, else the simplified points; the clouds as given
        without a sampler), or with sampled=False of the complete clouds.  Eval mode is the caller's."""
        out = []
        for s, e in _chunks(point_clouds.shape[0], batch_size):
            pc = point_clouds[s:e].contiguous()
            if sampled and self.sampler is not None:
                c = self._clouds.clouds(pc)
                pc = c["sampled"] if self.match_output else c["simplified"]
            out.append(self.classifier(pc)[1]["retrieval_vectors"])
        return torch.cat(out)

    def evaluate(self, point_clouds, labels, batch_size=32, database="sampled", recall_levels=11):
        """point_clouds (n, N, 3) and labels (n,) on the device -> {"map", "precision" (recall_levels,), "recall_levels" (recall_levels,),
        "ap" (n,), "num_queries"} with numpy arrays.  database="sampled": leave-one-out among the sampled clouds' descriptors; "complete": the
        sampled clouds query the complete clouds' descriptors, each query's own cloud left out.  "map" and "precision" are means over the
        "num_queries" queries with a relevant result, in float64; "ap" is NaN for the others.  One host read-back."""
        if database not in ("sampled", "complete"):
            raise ValueError("database must be 'sampled' or 'complete', got %r" % (database,))
        labels = labels.to(point_clouds.device).long().reshape(-1)
        with eval_mode(self.sampler, self.classifier):
            q = self.descriptors(point_clouds, batch_size)
            if database == "sampled":
                metrics = ops.retrieval_metrics(q, labels, recall_levels=recall_levels)
            else:
                x = self.descriptors(point_clouds, batch_size, sampled=False)
                metrics = ops.retrieval_metrics(q, labels, x, labels, recall_levels=recall_levels, exclude_diagonal=True)
            means, count = _retrieval_means(metrics)
            packed = torch.cat([count.reshape(1), means, metrics["ap"]]).cpu().numpy()
        L = int(recall_levels)
        return {"map": float(packed[1]), "precision": packed[2:2 + L], "recall_levels": np.linspace(0.0, 1.0, L),
                "ap": packed[2 + L:], "num_queries": int(packed[0])}


# ----------------------------------------------------------------------------------------------------- reconstruction
class ReconstructionEvaluator:
    """reconstruction/sampler/evaluate_samplenet.py and evaluate_samplenet_progressive.py on device tensors.  `sampler`: a
    ReconstructionSampleNet or a baseline sampler with "bnc" shapes; `ae`: PointNetAE or FrozenPointNetAE; ae_loss "chamfer" or "emd"
    (pointnet_ae.py:113-124).  hard_projection is evaluate_samplenet.py's --hard_projection (default 1): it selects the projection
    get_sample returns when it does not complete by FPS; get_samples always completes (samplenet_pointnet_ae.py:489), so the matched sample
    does not depend on it, as in the reference.  Methods return device tensors and never synchronise; evaluate() reads back once."""

    def __init__(self, sampler, ae, ae_loss="chamfer", hard_projection=1):
        if ae_loss not in ("chamfer", "emd"):
            raise ValueError("ae_loss must be 'chamfer' or 'emd'")
        self.sampler, self.ae, self.ae_loss, self.hard_projection = sampler, ae, ae_loss, int(hard_projection)

    def get_sample(self, X, complete_fps=True):
        """samplenet_pointnet_ae.py:459-477 for one batch (eval mode is the caller's): (sampled points (B, M, 3), their indices (B, M))."""
        X = X.contiguous()
        generated, _ = _sampler_output(self.sampler(X))
        generated = generated.contiguous()
        _, idx, _, _ = ops.nn_distance_forward(generated, X)
        if complete_fps:
            pts, pts_idx, _ = sputils.simple_projection_and_continued_fps(X, generated, idx)
            return pts, pts_idx
        project = getattr(self.sampler, "project", None)
        if isinstance(project, tf_ops.SoftProjection):
            return project(X, generated, hard=bool(self.hard_projection))[0], idx
        return generated, idx

    def get_samples(self, pclouds, batch_size=50):
        """samplenet_pointnet_ae.py:479-492: (sampled_pc (n, M, 3), sample_idx (n, M) int32)."""
        with eval_mode(self.sampler):
            parts = [self.get_sample(pclouds[s:e]) for s, e in _chunks(pclouds.shape[0], batch_size)]
        return torch.cat([p for p, _ in parts]), torch.cat([i for _, i in parts])

    def get_reconstructions_from_sampled(self, sampled_pc, batch_size=50):
        """sampler_progressive_autoencoder.py:165-177: the AE's reconstruction of every sampled cloud."""
        with eval_mode(self.ae):
            return torch.cat([self.ae(sampled_pc[s:e].contiguous()) for s, e in _chunks(sampled_pc.shape[0], batch_size)])

    def _loss(self, recon, gt):
        """Per-cloud AE loss (pointnet_ae.py:113-124 at batch 1) of recon (P * B, n, 3) against gt (B, n, 3), repeating every B clouds."""
        if self.ae_loss == "chamfer":
            return ops.chamfer_per_cloud(recon.contiguous(), gt.contiguous()).sum(dim=1)
        if not ops.emd_exact_mode() and ops.emd_per_cloud_supported(recon, gt):
            return ops.emd_per_cloud(recon.contiguous(), gt.contiguous())
        gt = gt.repeat(recon.shape[0] // gt.shape[0], 1, 1) if recon.shape[0] != gt.shape[0] else gt
        return tf_ops.match_cost(recon, gt, tf_ops.approx_match(recon, gt))

    def get_loss_ae_per_pc(self, pclouds, sampled_pc=None, batch_size=50):
        """sampler_progressive_autoencoder.py:145-163 without its loop over single clouds: the AE loss of every cloud's reconstruction from
        sampled_pc against the cloud, (n,).  sampled_pc=None reconstructs from the complete cloud: the reference loss of
        autoencoder/evaluate_ae.py that the NRE divides by."""
        feed = pclouds if sampled_pc is None else sampled_pc
        with eval_mode(self.ae):
            return torch.cat([self._loss(self.ae(feed[s:e].contiguous()), pclouds[s:e]) for s, e in _chunks(pclouds.shape[0], batch_size)])

    def get_loss_ae_per_pc_progressive(self, pclouds, sampled_pc, sizes, batch_size=50):
        """The AE loss of the reconstruction from sampled_pc[:, :s] for every s in sizes, (len(sizes), n): what evaluate_samplenet_progressive.py
        computes one size per run.  An AE with prefixes() reconstructs 16 sizes per shared encoder pass, and with the Chamfer loss their
        P * B reconstructions meet the B input clouds in one chamfer_per_cloud launch."""
        sizes = [int(s) for s in sizes]
        if not sizes or min(sizes) < 1 or max(sizes) > sampled_pc.shape[1]:
            raise ValueError("sizes must lie in [1, %d]" % sampled_pc.shape[1])
        asc = sorted(set(sizes))
        cols = []
        with eval_mode(self.ae):
            for s, e in _chunks(pclouds.shape[0], batch_size):
                samp, gt = sampled_pc[s:e].contiguous(), pclouds[s:e]
                # a frozen wrapper's prefixes(); CudaPointNetAE keeps its per-size forward, as the reconstruction steps do by default
                if hasattr(self.ae, "prefixes") and not isinstance(self.ae, tasknets.CudaPointNetAE):
                    rows = [self._loss(self.ae.prefixes(samp, asc[i:i + PREFIX_CHUNK]).flatten(0, 1), gt).view(-1, e - s)
                            for i in range(0, len(asc), PREFIX_CHUNK)]
                    cols.append(torch.cat(rows))
                else:
                    cols.append(torch.stack([self._loss(self.ae(samp[:, :k].contiguous()), gt) for k in asc]))
        out = torch.cat(cols, dim=1)
        return out if asc == sizes else out[[asc.index(s) for s in sizes]]

    nre = staticmethod(nre)

    def evaluate(self, pclouds, sizes=None, batch_size=50):
        """One sampling pass and the curve: {"ae_loss_per_pc", "ae_loss_per_pc_ref", "nre_per_pc", "mean_ae_loss", "nre"} as numpy, per cloud
        (n,) for sizes=None (the sampler's own size, evaluate_samplenet.py:93-152) and (len(sizes), n) with "mean_ae_loss" and "nre" per
        size otherwise; plus "sampled_pc" and "sample_idx" on the device.  One host read-back."""
        sampled_pc, sample_idx = self.get_samples(pclouds, batch_size)
        if sizes is None:
            loss = self.get_loss_ae_per_pc(pclouds, sampled_pc, batch_size)[None]
        else:
            loss = self.get_loss_ae_per_pc_progressive(pclouds, sampled_pc, sizes, batch_size)
        ref = self.get_loss_ae_per_pc(pclouds, None, batch_size)
        both = torch.cat([loss, ref[None]]).cpu().numpy().astype(np.float64)
        loss, ref = both[:-1], both[-1]
        ratio = nre(loss, ref[None])
        out = {"ae_loss_per_pc": loss, "ae_loss_per_pc_ref": ref, "nre_per_pc": ratio, "mean_ae_loss": loss.mean(axis=1), "nre": ratio.mean(axis=1)}
        if sizes is None:
            out = {k: (v[0] if k != "ae_loss_per_pc_ref" else v) for k, v in out.items()}
        out.update({"sampled_pc": sampled_pc, "sample_idx": sample_idx})
        return out
