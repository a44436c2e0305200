"""Loss composition of the three reference trainers, restated over this package's API (SURVEY.md 8f rank 1: the callers).

Only the sampling-related step logic is here; the task networks (PCRNet, the PointNet classifier, the auto-encoder), their
optimisers and the data pipelines stay the reference's.  Every function takes the task-side quantities as arguments and returns
what the reference's step returns, so a maintainer can swap the body of the corresponding method for one call.

    registration    registration/main.py:500-538         compute_samplenet_loss
    classification  classification/train_samplenet.py:163-180
    reconstruction  reconstruction/src/pointnet_ae.py:110-124 (AE loss), samplenet_pointnet_ae.py:165-189 (simplification loss)
    progressive reconstruction  reconstruction/src/samplenet_progressive_pointnet_ae.py:46-220   ProgressiveReconstructionStep
    task networks   classification/train_classifier.py (ClassifierTrainStep), reconstruction/src/pointnet_ae.py (AutoencoderTrainStep)
"""
import torch

from . import tf_ops


def registration_samplenet_loss(sampler, p0, p1, num_out_points, alpha, lmbda, gamma=1, delta=0, num_sampled_clouds=1):
    """`Action.compute_samplenet_loss` (registration/main.py:500-538).  p0: template, p1: source, both in `sampler.input_shape`.
    Returns (samplenet_loss, (p0_out, p1_projected), info) with info = {"simplification_loss", "projection_loss"}."""
    if num_sampled_clouds not in (1, 2):
        raise ValueError("num_sampled_clouds must be 1 or 2")
    to_bnc = (lambda t: t) if sampler.input_shape == "bnc" else (lambda t: t.permute(0, 2, 1).contiguous())
    out_bnc = (lambda t: t) if sampler.output_shape == "bnc" else (lambda t: t.permute(0, 2, 1).contiguous())
    p1_simplified, p1_projected = sampler(p1)
    simplification_loss = sampler.get_simplification_loss(to_bnc(p1), out_bnc(p1_simplified), num_out_points, gamma, delta)
    p0_out = p0
    if num_sampled_clouds == 2:   # sample the template as well
        p0_simplified, p0_projected = sampler(p0)
        p0_loss = sampler.get_simplification_loss(to_bnc(p0), out_bnc(p0_simplified), num_out_points, gamma, delta)
        simplification_loss = 0.5 * (simplification_loss + p0_loss)
        p0_out = p0_projected
    projection_loss = sampler.get_projection_loss()
    samplenet_loss = alpha * simplification_loss + lmbda * projection_loss
    return samplenet_loss, (p0_out, p1_projected), {"simplification_loss": simplification_loss, "projection_loss": projection_loss}


def classification_total_loss(loss_classifier, point_clouds, simplified_points, num_out_points, alpha, lmbda, gamma, delta, loss_projection):
    """classification/train_samplenet.py:173-180: `loss_classifier + ALPHA * loss_simplification + LMBDA * loss_projection` with the
    TF model's `get_simplification_loss` (samplenet_model.py:176-188) on (B,N,3) clouds.  Returns (loss, loss_simplification)."""
    loss_simplification = tf_ops.get_simplification_loss(point_clouds, simplified_points, num_out_points, gamma, delta)
    return loss_classifier + alpha * loss_simplification + lmbda * loss_projection, loss_simplification


def autoencoder_loss(x_reconstr, gt, loss="chamfer"):
    """`PointNetAutoEncoder._create_loss` (reconstruction/src/pointnet_ae.py:113-124): Chamfer = mean(d12) + mean(d21) over the batch;
    EMD = mean over the batch of match_cost(x, gt, approx_match(x, gt))."""
    if loss == "chamfer":
        cost_p1_p2, _, cost_p2_p1, _ = tf_ops.nn_distance(x_reconstr, gt)
        return cost_p1_p2.mean() + cost_p2_p1.mean()
    if loss == "emd":
        match = tf_ops.approx_match(x_reconstr, gt)
        return tf_ops.match_cost(x_reconstr, gt, match).mean()
    raise ValueError("loss must be 'chamfer' or 'emd'")


def autoencoder_simplification_loss(ref_pc, samp_pc, pc_size, is_denoising=False):
    """`SampleNetPointNetAE._get_simplification_loss` (reconstruction/src/samplenet_pointnet_ae.py:165-189): weight w = pc_size / 64
    (doubled when denoising) on the input->sample term.  Returns (loss, dist, idx, dist2, nn_distance_per_cloud (B,1))."""
    cost_p1_p2, idx, cost_p2_p1, _ = tf_ops.nn_distance(samp_pc, ref_pc)
    max_cost = cost_p1_p2.max(dim=1)[0].mean()
    per_cloud = cost_p1_p2.mean(dim=1, keepdim=True) + cost_p2_p1.mean(dim=1, keepdim=True)
    w = pc_size / 64.0
    loss = cost_p1_p2.mean() + max_cost + (2 * w if is_denoising else w) * cost_p2_p1.mean()
    return loss, cost_p1_p2, idx, cost_p2_p1, per_cloud


def progressive_simplification_loss(ref_pc, ordered_samples, sizes, gamma=1, delta=0, one_pass=True):
    """SampleNetProgressive (classification/train_samplenet_progressive.py:196-220): the simplification loss summed over the
    prefixes `ordered_samples[:, :s]` for s in `sizes`.  one_pass=True (default): ONE launch evaluates every prefix (the sample -> input
    distances of a prefix are a slice, the input -> sample distances a running prefix minimum: csrc/progressive.cu); one_pass=False: the
    reference's structure, one Chamfer evaluation per prefix."""
    sizes = [int(s) for s in sizes]
    if one_pass and len(sizes) <= 16 and ordered_samples.shape[1] <= 4096 and sorted(set(sizes)) == sizes:
        from . import ops

        total, _ = ops.ProgressiveLossFunction.apply(ordered_samples, ref_pc, sizes, [gamma + delta * s for s in sizes])
        return total
    total = torch.zeros((), device=ref_pc.device)
    for s in sizes:
        total = total + tf_ops.get_simplification_loss(ref_pc, ordered_samples[:, :s].contiguous(), s, gamma, delta)
    return total


# ----------------------------------------------------------------------------------------------------- whole steps with task networks
class ClassificationStep:
    """One training step of classification/train_samplenet.py:154-199: sampler (generator + TF-flavoured soft projection, sigma = T^2) in
    front of a FROZEN PointNet classifier; loss = loss_classifier + ALPHA * loss_simplification + LMBDA * loss_projection.
    `sampler` is a SampleNet-like module returning (simplified, projected) on (B,N,3) input; `classifier` a tasknets.PointNetCls
    (pointnet_cls_basic.py), a tasknets.PointNetClsTransforms (pointnet_cls.py, the trainer's default), or one of their frozen CUDA wrappers."""

    def __init__(self, sampler, classifier, num_out_points, alpha=30.0, lmbda=1.0, gamma=1.0, delta=0.0):
        self.sampler, self.classifier = sampler, classifier
        self.M, self.alpha, self.lmbda, self.gamma, self.delta = num_out_points, alpha, lmbda, gamma, delta
        classifier.requires_grad_(False)
        classifier.eval()

    def loss(self, point_clouds, labels):
        simplified, projected = self.sampler(point_clouds)
        pred, end_points = self.classifier(projected)
        loss_classifier = self.classifier.get_loss(pred, labels, end_points)
        loss_simplification = self.sampler.get_simplification_loss(point_clouds, simplified, self.M, self.gamma, self.delta)
        loss_projection = self.sampler.get_projection_loss()
        total = loss_classifier + self.alpha * loss_simplification + self.lmbda * loss_projection
        return total, {"loss_classifier": loss_classifier, "loss_simplification": loss_simplification, "loss_projection": loss_projection, "pred": pred}


class ProgressiveClassificationStep(ClassificationStep):
    """classification/train_samplenet_progressive.py:156-230: ONE generator pass emits MAX ordered points; the classifier and the
    simplification loss are evaluated on every power-of-two prefix and summed."""

    def __init__(self, sampler, classifier, min_points, max_points, alpha=30.0, lmbda=1.0, gamma=1.0, delta=0.0):
        super().__init__(sampler, classifier, max_points, alpha, lmbda, gamma, delta)
        self.sizes = []
        s = min_points
        while s <= max_points:
            self.sizes.append(s)
            s *= 2

    def loss(self, point_clouds, labels):
        simplified, projected = self.sampler(point_clouds)
        loss_classifier = 0.0
        if hasattr(self.classifier, "prefixes"):   # a frozen wrapper (tasknets.FrozenPointNetCls[Transforms]): every prefix from one pass
            preds, end_points = self.classifier.prefixes(projected, self.sizes, return_end_points=True)
            for pred, ep in zip(preds, end_points):
                loss_classifier = loss_classifier + self.classifier.get_loss(pred, labels, ep)
        else:
            for s in self.sizes:
                pred, end_points = self.classifier(projected[:, :s].contiguous())
                loss_classifier = loss_classifier + self.classifier.get_loss(pred, labels, end_points)
        loss_simplification = progressive_simplification_loss(point_clouds, simplified, self.sizes, self.gamma, self.delta)
        loss_projection = self.sampler.get_projection_loss()
        total = loss_classifier + self.alpha * loss_simplification + self.lmbda * loss_projection
        return total, {"loss_classifier": loss_classifier, "loss_simplification": loss_simplification, "loss_projection": loss_projection}


class ReconstructionStep:
    """One training step of reconstruction/src/samplenet_pointnet_ae.py:46-189: sampler (rec widths, sigma = max(T, 1e-2)^2) in front of a
    FROZEN auto-encoder; loss = AE loss(reconstruction of the projected points, input cloud) [Chamfer or EMD] + ALPHA * simplification
    loss (weight pc_size / 64 on the input -> sample term) + LMBDA * projection loss."""

    def __init__(self, sampler, ae, num_out_points, alpha=0.01, lmbda=1e-4, ae_loss="chamfer"):
        self.sampler, self.ae, self.M, self.alpha, self.lmbda, self.ae_loss = sampler, ae, num_out_points, alpha, lmbda, ae_loss
        ae.requires_grad_(False)
        ae.eval()

    def loss(self, point_clouds):
        simplified, projected = self.sampler(point_clouds)
        x_reconstr = self.ae(projected)
        loss_ae = autoencoder_loss(x_reconstr, point_clouds, self.ae_loss)
        loss_simplification, _, _, _, _ = autoencoder_simplification_loss(point_clouds, simplified, self.M)
        loss_projection = self.sampler.get_projection_loss()
        total = loss_ae + self.alpha * loss_simplification + self.lmbda * loss_projection
        return total, {"loss_ae": loss_ae, "loss_simplification": loss_simplification, "loss_projection": loss_projection}


class ProgressiveReconstructionStep:
    """One training step of reconstruction/src/samplenet_progressive_pointnet_ae.py:46-220 (the progressive reconstruction trainer,
    reconstruction/sampler/train_samplenet_progressive.py): ONE sampler pass emits max(sizes) ordered points, projected with the
    reconstruction SoftProjection; for every prefix s the FROZEN auto-encoder reconstructs projected[:, :s], and
    loss = mean over prefixes of the Chamfer AE loss + ALPHA * mean over prefixes of the simplification loss of simplified[:, :s]
    (weight s / 64 on the input -> sample term) + LMBDA * projection loss.

    Only the Chamfer AE loss is restated: the reference's EMD branch (:158-160) matches against `self.x_reconstr`, which :102 assigns only
    after the loop, so its progressive graph builds with Chamfer alone; ae_loss="emd" raises ValueError."""

    def __init__(self, sampler, ae, sizes=(16, 32, 64, 128, 256, 512, 1024, 2048), alpha=0.01, lmbda=1e-4, ae_loss="chamfer"):
        if ae_loss != "chamfer":
            raise ValueError("the progressive reconstruction step has a Chamfer AE loss only (the reference's EMD branch does not build)")
        self.sampler, self.ae, self.alpha, self.lmbda = sampler, ae, alpha, lmbda
        self.sizes = [int(s) for s in sizes]
        ae.requires_grad_(False)
        ae.eval()

    def loss(self, point_clouds):
        simplified, projected = self.sampler(point_clouds)
        # one Chamfer evaluation over every prefix's reconstruction: equal-size terms, so the mean over all of them is the mean over prefixes
        if hasattr(self.ae, "prefixes"):   # a frozen wrapper (tasknets.FrozenPointNetAE): every prefix from one shared pass
            x_reconstr = self.ae.prefixes(projected, self.sizes).flatten(0, 1)
        else:
            x_reconstr = torch.cat([self.ae(projected[:, :s].contiguous()) for s in self.sizes])
        loss_ae = autoencoder_loss(x_reconstr, point_clouds.repeat(len(self.sizes), 1, 1))
        loss_simplification = progressive_simplification_loss(point_clouds, simplified, self.sizes, gamma=0, delta=1 / 64.0) / len(self.sizes)
        loss_projection = self.sampler.get_projection_loss()
        total = loss_ae + self.alpha * loss_simplification + self.lmbda * loss_projection
        return total, {"loss_ae": loss_ae, "loss_simplification": loss_simplification, "loss_projection": loss_projection}


# ----------------------------------------------------------------------------------------------------- training the task networks
def staircase_decay(base, step, decay_step, decay_rate):
    """tf.train.exponential_decay(base, step, decay_step, decay_rate, staircase=True): base * decay_rate ** floor(step / decay_step)."""
    return base * decay_rate ** (step // decay_step)


class ClassifierTrainStep:
    """One training step of classification/train_classifier.py:104-240 on a PointNet classifier (tasknets.PointNetCls,
    PointNetClsTransforms, or a wrapper with the module's forward and get_loss).  Step s (counted from 0, `self.step`) uses

        learning rate  max(staircase_decay(base_lr, s * batch_size, decay_step, decay_rate), 1e-5)     (get_learning_rate)
        BatchNorm      bn_decay = min(0.99, 1 - staircase_decay(0.5, s * batch_size, decay_step, 0.5)) (get_bn_decay), applied as torch
                       momentum 1 - bn_decay on every BatchNorm of the network

    then runs get_loss, backward and optimizer.step().  __call__(points (B, N, 3), labels (B,)) -> (loss, pred (B,) int64, correct)."""

    def __init__(self, net, optimizer, batch_size=32, base_lr=1e-3, decay_step=200000, decay_rate=0.7):
        self.net, self.optimizer = net, optimizer
        self.batch_size, self.base_lr, self.decay_step, self.decay_rate = batch_size, base_lr, decay_step, decay_rate
        self.step = 0

    def learning_rate(self, step):
        return max(staircase_decay(self.base_lr, step * self.batch_size, self.decay_step, self.decay_rate), 1e-5)

    def bn_decay(self, step):
        return min(0.99, 1.0 - staircase_decay(0.5, step * self.batch_size, float(self.decay_step), 0.5))

    def __call__(self, points, labels):
        lr, momentum = self.learning_rate(self.step), 1.0 - self.bn_decay(self.step)
        for g in self.optimizer.param_groups:
            g["lr"] = lr
        for m in self.net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.momentum = momentum
        self.net.train()
        self.optimizer.zero_grad()
        logits, end_points = self.net(points)
        loss = self.net.get_loss(logits, labels, end_points)
        loss.backward()
        self.optimizer.step()
        self.step += 1
        pred = logits.detach().argmax(dim=1)
        return loss.detach(), pred, int((pred == labels.long()).sum())


class AutoencoderTrainStep:
    """One training step of the point-cloud autoencoder (reconstruction/src/pointnet_ae.py:46-56, 110-150) on tasknets.PointNetAE or
    tasknets.CudaPointNetAE: the input is the first n_sample_points points of each cloud, or with use_fps their farthest point sample
    (ops.farthest_point_sample); loss = autoencoder_loss(reconstruction, gt) with Chamfer or EMD; backward; optimizer.step().  The learning
    rate is the optimiser's.  __call__(x (B, N, 3), gt=None (x)) -> loss."""

    def __init__(self, ae, optimizer, ae_loss="chamfer", use_fps=False, n_sample_points=2048):
        if ae_loss not in ("chamfer", "emd"):
            raise ValueError("ae_loss must be 'chamfer' or 'emd'")
        self.ae, self.optimizer, self.ae_loss, self.use_fps, self.n_sample_points = ae, optimizer, ae_loss, use_fps, n_sample_points

    def __call__(self, x, gt=None):
        gt = x if gt is None else gt
        if self.use_fps:
            from . import ops

            _, s = ops.farthest_point_sample(x.contiguous(), self.n_sample_points, return_points=True)
        else:
            s = x[:, :self.n_sample_points].contiguous()
        self.ae.train()
        self.optimizer.zero_grad()
        loss = autoencoder_loss(self.ae(s), gt, self.ae_loss)
        loss.backward()
        self.optimizer.step()
        return loss.detach()
