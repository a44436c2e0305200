"""Loss composition of the three reference trainers, restated over this package's API (SURVEY.md 8f rank 1: the callers).

Only the sampling-related step logic is here; the task networks (PCRNet, the PointNet classifier, the auto-encoder), their
optimisers and the data pipelines stay the reference's.  Every function takes the task-side quantities as arguments and returns
what the reference's step returns, so a maintainer can swap the body of the corresponding method for one call.

    registration    registration/main.py:500-538         compute_samplenet_loss
    classification  classification/train_samplenet.py:163-180
    reconstruction  reconstruction/src/pointnet_ae.py:110-124 (AE loss), samplenet_pointnet_ae.py:165-189 (simplification loss)
    progressive reconstruction  reconstruction/src/samplenet_progressive_pointnet_ae.py:46-220   ProgressiveReconstructionStep
    task networks   classification/train_classifier.py (ClassifierTrainStep), reconstruction/src/pointnet_ae.py (AutoencoderTrainStep)
    sampler epochs  the four SampleNet training scripts around the steps above (SamplerTrainStep)
"""
import torch

from . import tasknets, tf_ops


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
    EMD = mean over the batch of match_cost(x, gt, approx_match(x, gt)); inside its envelope through ops.EMDCostFunction in the mode
    approx_match would take (fast, or exact with SNB200_EMD_EXACT_EXP=1), which gives the same cost and gradients bit for bit without the
    (B, N, N) match tensor."""
    if loss == "chamfer":
        cost_p1_p2, _, cost_p2_p1, _ = tf_ops.nn_distance(x_reconstr, gt)
        return cost_p1_p2.mean() + cost_p2_p1.mean()
    if loss == "emd":
        from . import ops

        exact = ops.emd_exact_mode()
        if x_reconstr.shape[0] == gt.shape[0] and ops.emd_per_cloud_supported(x_reconstr, gt, exact):
            return ops.EMDCostFunction.apply(x_reconstr, gt, exact).mean()
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


def _fix_or_check_ae(ae, fixed_ae, ae_batch_stats):
    """The reconstruction steps' fixed_ae: True freezes the auto-encoder (requires_grad_(False), eval mode); False checks that it can be
    trained and leaves it alone.  Returns the flag."""
    if fixed_ae:
        ae.requires_grad_(False)
        ae.eval()
        return True
    if isinstance(ae, tasknets.FrozenPointNetAE):
        raise ValueError("fixed_ae=False trains the auto-encoder: a FrozenPointNetAE cannot train (use tasknets.CudaPointNetAE or the module)")
    if ae_batch_stats:
        raise ValueError("fixed_ae=False runs the auto-encoder in training mode, which already normalises with the batch statistics: "
                         "ae_batch_stats=True is for the frozen auto-encoder")
    return False


class ReconstructionStep:
    """One training step of reconstruction/src/samplenet_pointnet_ae.py:46-189: sampler (rec widths, sigma = max(T, 1e-2)^2) in front of a
    FROZEN auto-encoder; loss = AE loss(reconstruction of the projected points, input cloud) [Chamfer or EMD] + ALPHA * simplification
    loss (weight pc_size / 64 on the input -> sample term) + LMBDA * projection loss.

    ae_batch_stats=True: the frozen auto-encoder normalises every BatchNorm with the batch statistics of the projected points, as the
    reference's trainer does (it runs the AE under tflearn's training flag with every moving-average decay at 1, so the AE's state never
    changes): the AE is called as ae(projected, batch_stats=True).  False (default): eval-mode BatchNorm from the running statistics, and the
    call takes no keyword, so any module works.

    fixed_ae=False (the reference's --fixed_ae False): the auto-encoder is trained together with the sampler.  The constructor leaves its
    requires_grad and mode alone, loss() puts it in training mode (BatchNorm over the batch, running statistics moving), and the optimiser
    may hold its parameters.  A tasknets.CudaPointNetAE runs as ae.prefixes(projected, [M])[0] (the batch-statistics encoder trained,
    see CudaPointNetAE.prefixes), any other module as ae(projected).  A FrozenPointNetAE (it cannot train) and ae_batch_stats=True
    (training mode already normalises with the batch statistics) raise ValueError."""

    def __init__(self, sampler, ae, num_out_points, alpha=0.01, lmbda=1e-4, ae_loss="chamfer", ae_batch_stats=False, fixed_ae=True):
        self.sampler, self.ae, self.M, self.alpha, self.lmbda, self.ae_loss = sampler, ae, num_out_points, alpha, lmbda, ae_loss
        self.ae_batch_stats = bool(ae_batch_stats)
        self.fixed_ae = _fix_or_check_ae(ae, fixed_ae, self.ae_batch_stats)

    def loss(self, point_clouds):
        simplified, projected = self.sampler(point_clouds)
        if not self.fixed_ae:
            self.ae.train()
            if isinstance(self.ae, tasknets.CudaPointNetAE):
                x_reconstr = self.ae.prefixes(projected, [projected.shape[1]])[0]
            else:
                x_reconstr = self.ae(projected)
        else:
            x_reconstr = self.ae(projected, batch_stats=True) if self.ae_batch_stats else self.ae(projected)
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
    after the loop, so its progressive graph builds with Chamfer alone; ae_loss="emd" raises ValueError.

    ae_batch_stats=True: every prefix is normalised with its own batch statistics, as the reference, which rebuilds the encoder per prefix
    under the training flag (see ReconstructionStep): ae.prefixes(projected, sizes, batch_stats=True), or ae(prefix, batch_stats=True) per
    prefix on a module without `prefixes`.

    fixed_ae=False: the auto-encoder is trained together with the sampler, as in ReconstructionStep; every prefix is normalised with its
    own batch statistics, and the running statistics move once per prefix in ascending order.  A tasknets.CudaPointNetAE runs as
    ae.prefixes(projected, sizes) (every prefix from one encoder pass), any other module as the ascending loop of ae(projected[:, :s])."""

    def __init__(self, sampler, ae, sizes=(16, 32, 64, 128, 256, 512, 1024, 2048), alpha=0.01, lmbda=1e-4, ae_loss="chamfer",
                 ae_batch_stats=False, fixed_ae=True):
        if ae_loss != "chamfer":
            raise ValueError("the progressive reconstruction step has a Chamfer AE loss only (the reference's EMD branch does not build)")
        self.sampler, self.ae, self.alpha, self.lmbda = sampler, ae, alpha, lmbda
        self.ae_batch_stats = bool(ae_batch_stats)
        self.sizes = [int(s) for s in sizes]
        self.fixed_ae = _fix_or_check_ae(ae, fixed_ae, self.ae_batch_stats)

    def loss(self, point_clouds):
        simplified, projected = self.sampler(point_clouds)
        # one Chamfer evaluation over every prefix's reconstruction: equal-size terms, so the mean over all of them is the mean over prefixes
        kw = {"batch_stats": True} if self.ae_batch_stats else {}
        if not self.fixed_ae:
            self.ae.train()
            if isinstance(self.ae, tasknets.CudaPointNetAE):
                x_reconstr = self.ae.prefixes(projected, self.sizes).flatten(0, 1)
            else:
                x_reconstr = torch.cat([self.ae(projected[:, :s].contiguous()) for s in self.sizes])
        elif hasattr(self.ae, "prefixes") and not isinstance(self.ae, tasknets.CudaPointNetAE):
            # a frozen wrapper (tasknets.FrozenPointNetAE): every prefix from one shared pass
            x_reconstr = self.ae.prefixes(projected, self.sizes, **kw).flatten(0, 1)
        else:
            x_reconstr = torch.cat([self.ae(projected[:, :s].contiguous(), **kw) for s in self.sizes])
        loss_ae = autoencoder_loss(x_reconstr, point_clouds.repeat(len(self.sizes), 1, 1))
        loss_simplification = progressive_simplification_loss(point_clouds, simplified, self.sizes, gamma=0, delta=1 / 64.0) / len(self.sizes)
        loss_projection = self.sampler.get_projection_loss()
        total = loss_ae + self.alpha * loss_simplification + self.lmbda * loss_projection
        return total, {"loss_ae": loss_ae, "loss_simplification": loss_simplification, "loss_projection": loss_projection}


# ----------------------------------------------------------------------------------------------------- training the task networks
def staircase_decay(base, step, decay_step, decay_rate):
    """tf.train.exponential_decay(base, step, decay_step, decay_rate, staircase=True): base * decay_rate ** floor(step / decay_step)."""
    return base * decay_rate ** (step // decay_step)


def pointnet_learning_rate(step, batch_size, base_lr, decay_step, decay_rate):
    """get_learning_rate of the PointNet classification scripts (train_classifier.py, train_samplenet.py, train_samplenet_progressive.py) at
    step `step` counted from 0: max(staircase_decay(base_lr, step * batch_size, decay_step, decay_rate), 1e-5)."""
    return max(staircase_decay(base_lr, step * batch_size, decay_step, decay_rate), 1e-5)


def pointnet_bn_decay(step, batch_size, decay_step):
    """get_bn_decay of the same scripts: min(0.99, 1 - staircase_decay(0.5, step * batch_size, decay_step, 0.5)); torch's BatchNorm momentum
    is 1 - bn_decay."""
    return min(0.99, 1.0 - staircase_decay(0.5, step * batch_size, float(decay_step), 0.5))


def _set_schedule(optimizer, lr, module, momentum):
    """The step's learning rate on every parameter group and, unless momentum is None, BatchNorm momentum on every BatchNorm1d of module."""
    for g in optimizer.param_groups:
        g["lr"] = lr
    if momentum is not None:
        for m in module.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.momentum = momentum


def _augment(points, gauss_augment, z_rotate):
    """general_utils.apply_augmentations on the device (ops.ae_augment); the batch itself when both are off (no launch)."""
    if gauss_augment is None and not z_rotate:
        return points
    from . import ops

    g = gauss_augment or {}
    return ops.ae_augment(points, g.get("mu"), g.get("sigma"), z_rotate)


def _check_augment(gauss_augment):
    if gauss_augment is not None and not (isinstance(gauss_augment, dict) and "mu" in gauss_augment and gauss_augment.get("sigma") is not None):
        raise ValueError("gauss_augment must be None or a dict with 'mu' and 'sigma', got %r" % (gauss_augment,))


def _epoch_batches(points, batch_size):
    """A fresh device permutation of the set's n clouds, split into n // batch_size whole batches of indices; the remainder is not used."""
    n = points.shape[0]
    steps = n // batch_size
    if steps < 1:
        raise ValueError("an epoch needs at least one whole batch of %d clouds, got %d" % (batch_size, n))
    perm = torch.randperm(n, device=points.device)
    return [perm[s * batch_size:(s + 1) * batch_size] for s in range(steps)]


def _step_sums(values, skip_last=False):
    """The float64 vector an epoch adds up for one step.  skip_last: the last value is the step's 0/1 skip flag, and a skipped step adds
    nothing but that flag (by select: its terms may be NaN)."""
    v = torch.stack([t.double() for t in values])
    if not skip_last:
        return v
    return torch.cat([v[:-1].masked_fill(values[-1].bool(), 0.0), v[-1:]])


def _mean_over(total, taken):
    """A mean over the steps taken: NaN when every step of the epoch was skipped."""
    return total / taken if taken else float("nan")


class _SkipNonfinite:
    """skip_nonfinite=True of the training runners.  begin() before the step copies every parameter and buffer of the trained modules and
    every optimiser state tensor into snapshot buffers made once (torch._foreach_copy_ per dtype); end(terms) after it runs ops.NonfiniteGuard over
    the step's floating terms, the optimiser's gradients and the modules' parameters and floating buffers, which copies the snapshots back
    when any of them holds a NaN or an Inf.  Optimiser state the step created (a parameter's first step) comes back as zeros, the fresh state
    of graphs.ZERO_INIT_OPTIMIZERS: skip_nonfinite needs one of them with capturable=True (a non-capturable Adam keeps its step count on
    the host, out of the guard's reach).  Everything stays on the device, in eager mode and inside a captured graph alike."""

    def __init__(self, modules, optimizer, who):
        from . import graphs, ops

        graphs.check_capturable(optimizer, who)
        self.optimizer = optimizer
        self.tensors = []
        for t in [t for m in modules for t in list(m.parameters()) + list(m.buffers())]:
            if all(t is not u for u in self.tensors):
                self.tensors.append(t)
        self.checked = [t for t in self.tensors if t.is_floating_point()]
        self.guard = ops.NonfiniteGuard(self.tensors[0].device)
        self.snap = {}                 # id(live tensor) -> (live, snapshot)
        self.key, self.copies = None, []

    def _params(self):
        return [p for g in self.optimizer.param_groups for p in g["params"]]

    def _live(self):
        state = [v for p in self._params() for v in self.optimizer.state.get(p, {}).values() if torch.is_tensor(v)]
        return self.tensors + state

    def begin(self):
        live = self._live()
        key = tuple(id(t) for t in live)
        if key != self.key:
            for t in live:
                if id(t) not in self.snap:
                    self.snap[id(t)] = (t, torch.empty_like(t))
            groups = {}                        # one multi-tensor copy per dtype: a mixed list falls back to a copy per tensor
            for t in live:
                dst, src = groups.setdefault(t.dtype, ([], []))
                dst.append(self.snap[id(t)][1])
                src.append(t)
            self.key, self.copies = key, list(groups.values())
        with torch.no_grad():
            for dst, src in self.copies:
                torch._foreach_copy_(dst, src)

    def end(self, terms):
        """The guard after the step; returns the step's skip flag (0/1 int32 device tensor, a copy)."""
        live = self._live()
        for t in live:                         # state this step created: restored as zeros
            if id(t) not in self.snap:
                self.snap[id(t)] = (t, torch.zeros_like(t))
        grads = [p.grad for p in self._params() if p.grad is not None]
        checked = [t for t in terms if t.is_floating_point()] + grads + self.checked
        return self.guard(checked, live, [self.snap[id(t)][1] for t in live]).clone()


class _StepGraph:
    """The CUDA-graph side of a runner built with graphed=True (the runners here and registration.RegistrationStep): static input buffers of
    one shape, a float64 accumulator of the step's terms, and the step captured (graphs.CapturedStep) at one schedule.

    `step(*inputs) -> (result, terms)` is the runner's step without its counters; the graph runs it on the static inputs and adds
    torch.stack(terms) in float64 to the accumulator.  replay(key) captures again, freeing the old graph first, whenever `key` (the
    schedule's frozen scalars: learning rates, BatchNorm momentum) differs from the captured one."""

    def __init__(self, owner, step, modules, optimizer, counters, skip_last=False):
        self.owner, self.step, self.modules, self.optimizer, self.counters = owner, step, modules, optimizer, counters
        self.skip_last = skip_last
        self.inputs, self.acc, self.key, self.captured = None, None, None, None

    def _check(self, shapes, tensors):
        """ValueError unless every input has its static buffer's shape, dtype and device: the runner holds one captured input."""
        for shape, t, s in zip(shapes, tensors, self.inputs):
            if tuple(shape) != tuple(s.shape) or t.dtype != s.dtype or t.device != s.device:
                raise ValueError("%s(graphed=True) holds one captured input: %s %s on %s; got %s %s on %s (build another runner for "
                                 "another one)" % (type(self.owner).__name__, tuple(s.shape), s.dtype, s.device, tuple(shape), t.dtype,
                                                   t.device))

    def bind(self, *tensors):
        """Copy the inputs into the static buffers (made on the first call); another shape, dtype or device raises ValueError."""
        if self.inputs is None:
            self.inputs = [torch.empty(t.shape, dtype=t.dtype, device=t.device) for t in tensors]
        self._check([t.shape for t in tensors], tensors)
        for s, t in zip(self.inputs, tensors):
            s.copy_(t)

    def select(self, sources, idx):
        """The batch `idx` of device-resident sets into the static buffers (made on the first call); the checks of bind."""
        if self.inputs is None:
            self.bind(*[src[idx] for src in sources])
            return
        self._check([(idx.numel(),) + tuple(src.shape[1:]) for src in sources], sources)
        for s, src in zip(self.inputs, sources):
            torch.index_select(src, 0, idx, out=s)

    def _body(self):
        result, terms = self.step(*self.inputs)
        v = _step_sums(terms, self.skip_last)
        if self.acc is None:   # the first warm-up of the first capture; the epoch zeroes it before its first replay
            self.acc = torch.zeros_like(v)
        self.acc += v
        return result

    def replay(self, key, first_of_epoch=False):
        """One step on the static inputs; returns the step's result (static buffers).  first_of_epoch zeroes the accumulator first."""
        if self.captured is None or key != self.key:
            from . import graphs

            self.captured = None
            self.captured = graphs.CapturedStep(self._body, self.modules, self.optimizer, counters=(self.owner, self.counters),
                                                state=[] if self.acc is None else [self.acc])
            self.key = key
        if first_of_epoch:
            self.acc.zero_()
        self.captured.replay()
        return self.captured.outputs


class ClassifierTrainStep:
    """One training step of classification/train_classifier.py:104-240 on a PointNet classifier (tasknets.PointNetCls,
    PointNetClsTransforms, or a wrapper with the module's forward and get_loss).  Step s (counted from 0, `self.step`) uses

        learning rate  max(staircase_decay(base_lr, s * batch_size, decay_step, decay_rate), 1e-5)     (get_learning_rate)
        BatchNorm      bn_decay = min(0.99, 1 - staircase_decay(0.5, s * batch_size, decay_step, 0.5)) (get_bn_decay), applied as torch
                       momentum 1 - bn_decay on every BatchNorm of the network

    then runs get_loss, backward and optimizer.step().  __call__(points (B, N, 3), labels (B,)) -> (loss, pred (B,) int64, correct).

    augment=True feeds the network the reference's augmented batch (train_classifier.py:217-221): ops.rotate_jitter(points, sigma, clip), a
    random rotation about the up axis per cloud, then the clipped jitter, on the device.  Its key is drawn from torch's default CUDA
    generator before the forward, so before the dropout masks of the CUDA wrappers.  augment=False (default) feeds the batch as it is.

    graphed=True runs every step as one CUDA-graph replay (see SamplerTrainStep): the same results bit for bit, loss and pred as static
    buffers.  It needs a capturable optimizer of graphs.ZERO_INIT_OPTIMIZERS and holds one (B, N).

    skip_nonfinite=True skips a step that goes non-finite, as SamplerTrainStep does: __call__ returns (loss, pred, correct, skipped) and
    train_one_epoch adds "skipped_steps", its means taken over the steps not skipped."""

    def __init__(self, net, optimizer, batch_size=32, base_lr=1e-3, decay_step=200000, decay_rate=0.7, augment=False, sigma=0.01, clip=0.05,
                 graphed=False, skip_nonfinite=False):
        if augment and not (sigma >= 0 and clip > 0):
            raise ValueError("augmentation needs sigma >= 0 and clip > 0 (sigma=%r clip=%r)" % (sigma, clip))
        self.net, self.optimizer = net, optimizer
        self.batch_size, self.base_lr, self.decay_step, self.decay_rate = batch_size, base_lr, decay_step, decay_rate
        self.augment, self.sigma, self.clip = bool(augment), float(sigma), float(clip)
        self.step = 0
        self.graphed = bool(graphed)
        if self.graphed:
            from .graphs import check_capturable

            check_capturable(optimizer, type(self).__name__ + "(graphed=True)")
        self._skip = _SkipNonfinite([net], optimizer, type(self).__name__ + "(skip_nonfinite=True)") if skip_nonfinite else None
        self._graph = _StepGraph(self, self._step, [net], optimizer, ("step",), self._skip is not None) if self.graphed else None

    def learning_rate(self, step):
        return pointnet_learning_rate(step, self.batch_size, self.base_lr, self.decay_step, self.decay_rate)

    def bn_decay(self, step):
        return pointnet_bn_decay(step, self.batch_size, self.decay_step)

    def _schedule(self):
        """Set the schedule of step self.step; returns its (learning rate, BatchNorm momentum)."""
        lr, momentum = self.learning_rate(self.step), 1.0 - self.bn_decay(self.step)
        _set_schedule(self.optimizer, lr, self.net, momentum)
        return lr, momentum

    def _step(self, points, labels):
        """One step without the step count: ((loss, pred, correct) as device tensors, the terms an epoch sums)."""
        self._schedule()
        if self._skip is not None:
            self._skip.begin()
        if self.augment:
            from . import ops

            points = ops.rotate_jitter(points, self.sigma, self.clip)
        self.net.train()
        self.optimizer.zero_grad()
        logits, end_points = self.net(points)
        loss = self.net.get_loss(logits, labels, end_points)
        loss.backward()
        self.optimizer.step()
        pred = logits.detach().argmax(dim=1)
        correct = (pred == labels.long()).sum()
        if self._skip is None:
            return (loss.detach(), pred, correct), (loss.detach(), correct)
        skipped = self._skip.end([loss.detach()])
        return (loss.detach(), pred, correct, skipped), (loss.detach(), correct, skipped)

    def _run(self, points, labels, first_of_epoch=False):
        """One step; (loss, pred, correct) as device tensors, without a host synchronisation.  Graphed: a replay on the bound inputs."""
        out = self._graph.replay(self._schedule(), first_of_epoch) if self.graphed else self._step(points, labels)[0]
        self.step += 1
        return out

    def __call__(self, points, labels):
        if self.graphed:
            self._graph.bind(points, labels)
        out = self._run(points, labels)
        return (out[0], out[1], int(out[2])) + tuple(out[3:])

    def train_one_epoch(self, points, labels):
        """train_one_epoch (train_classifier.py:185-242) over one device-resident set, points (n, N, 3) and labels (n,): shuffle with
        torch.randperm on the device, run n // batch_size whole batches (the remainder is not used, as in the reference), accumulate the loss
        sum in float64 and the correct count on the device, and read them back once.  -> {"mean_loss", "accuracy", "steps"}, and
        "skipped_steps" with skip_nonfinite, the means then over the steps taken (NaN if none was)."""
        batches = _epoch_batches(points, self.batch_size)
        steps = len(batches)
        labels = labels.to(points.device).reshape(-1)
        if self.graphed:
            for s, idx in enumerate(batches):
                self._graph.select((points, labels), idx)
                self._run(None, None, first_of_epoch=s == 0)
            host = self._graph.acc.cpu()
        elif self._skip is None:
            loss_sum = torch.zeros((), dtype=torch.float64, device=points.device)
            correct = torch.zeros((), dtype=torch.int64, device=points.device)
            for idx in batches:
                loss, _, c = self._run(points[idx], labels[idx])
                loss_sum += loss.double()
                correct += c
            host = torch.stack([loss_sum, correct.double()]).cpu()
        else:
            sums = torch.zeros(3, dtype=torch.float64, device=points.device)
            for idx in batches:
                loss, _, c, skipped = self._run(points[idx], labels[idx])
                sums += _step_sums([loss, c, skipped], True)
            host = sums.cpu()
        if self._skip is None:
            return {"mean_loss": float(host[0]) / steps, "accuracy": float(host[1]) / (steps * self.batch_size), "steps": steps}
        taken = steps - int(host[2])
        return {"mean_loss": _mean_over(float(host[0]), taken), "accuracy": _mean_over(float(host[1]), taken * self.batch_size), "steps": steps,
                "skipped_steps": steps - taken}


class AutoencoderTrainStep:
    """One training step of the point-cloud autoencoder (reconstruction/src/pointnet_ae.py:46-56, 110-150) on tasknets.PointNetAE or
    tasknets.CudaPointNetAE: the input is the first n_sample_points points of each cloud, or with use_fps their farthest point sample
    (ops.farthest_point_sample); loss = autoencoder_loss(reconstruction, gt) with Chamfer or EMD; backward; optimizer.step().  The learning
    rate is the optimiser's.  __call__(x (B, N, 3), gt=None) -> loss.

    gauss_augment (None or {"mu", "sigma"}) and z_rotate are the configuration's augmentation (train_ae.py; off by default, as in
    ae_templates.default_train_params): __call__ first replaces x by ops.ae_augment(x, mu, sigma, z_rotate), as _single_epoch_train applies
    general_utils.apply_augmentations to every batch.  gt=None scores against that augmented batch, or with denoising=True (train_ae.py:105)
    against the batch as given (pointnet_ae.py:168-183).  With both off no launch is added.  batch_size is train_one_epoch's.

    graphed=True runs every step as one CUDA-graph replay (see SamplerTrainStep), the loss a static buffer; a change of the optimiser's
    learning rates captures again.  It needs a capturable optimizer of graphs.ZERO_INIT_OPTIMIZERS, holds one (B, N) and takes no gt.

    skip_nonfinite=True skips a step that goes non-finite, as SamplerTrainStep does: __call__ returns (loss, skipped) and train_one_epoch
    adds "skipped_steps", its loss the mean over the steps not skipped."""

    def __init__(self, ae, optimizer, ae_loss="chamfer", use_fps=False, n_sample_points=2048, batch_size=50, gauss_augment=None, z_rotate=False,
                 denoising=False, graphed=False, skip_nonfinite=False):
        if ae_loss not in ("chamfer", "emd"):
            raise ValueError("ae_loss must be 'chamfer' or 'emd'")
        _check_augment(gauss_augment)
        self.ae, self.optimizer, self.ae_loss, self.use_fps, self.n_sample_points = ae, optimizer, ae_loss, use_fps, n_sample_points
        self.batch_size, self.gauss_augment, self.z_rotate, self.denoising = batch_size, gauss_augment, bool(z_rotate), bool(denoising)
        self.graphed = bool(graphed)
        if self.graphed:
            from .graphs import check_capturable

            check_capturable(optimizer, type(self).__name__ + "(graphed=True)")
        self._skip = _SkipNonfinite([ae], optimizer, type(self).__name__ + "(skip_nonfinite=True)") if skip_nonfinite else None
        self._graph = _StepGraph(self, self._graph_step, [ae], optimizer, (), self._skip is not None) if self.graphed else None

    def _graph_step(self, x):
        out = self._step(x)
        return out, (list(out) if self._skip is not None else [out])

    def _replay(self, first_of_epoch=False):
        return self._graph.replay(tuple(g["lr"] for g in self.optimizer.param_groups), first_of_epoch)

    def __call__(self, x, gt=None):
        if not self.graphed:
            return self._step(x, gt)
        if gt is not None:
            raise ValueError("AutoencoderTrainStep(graphed=True) scores against its own batch (gt=None); build it with graphed=False for a gt")
        self._graph.bind(x)
        return self._replay()

    def _step(self, x, gt=None):
        if self._skip is not None:
            self._skip.begin()
        aug = _augment(x, self.gauss_augment, self.z_rotate)
        gt = (x if self.denoising else aug) if gt is None else gt
        x = aug
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
        if self._skip is None:
            return loss.detach()
        return loss.detach(), self._skip.end([loss.detach()])

    def train_one_epoch(self, points):
        """_single_epoch_train (reconstruction/src/pointnet_ae.py:153-194) over one device-resident set points (n, N, 3): shuffle with
        torch.randperm on the device, run n // batch_size whole batches through __call__ (augmented as configured; with denoising the clean
        batch is the target), sum the losses in float64 on the device and read the sum back once.  in_out.PointCloudDataSet.next_batch
        (in_out.py:350-370) reshuffles when a batch would run past the end, so with int(n / batch_size) batches per epoch every epoch is a
        fresh permutation whose remainder is not used: the same epoch.  -> {"loss": mean over batches, divided by N with EMD, "steps"}, and
        "skipped_steps" with skip_nonfinite, the mean then over the steps taken (NaN if none was)."""
        batches = _epoch_batches(points, self.batch_size)
        skip = self._skip is not None
        if self.graphed:
            for s, idx in enumerate(batches):
                self._graph.select((points,), idx)
                self._replay(first_of_epoch=s == 0)
            sums = self._graph.acc
        elif not skip:
            sums = torch.zeros((), dtype=torch.float64, device=points.device)
            for idx in batches:
                sums += self(points[idx]).double()
        else:
            sums = torch.zeros(2, dtype=torch.float64, device=points.device)
            for idx in batches:
                sums += _step_sums(list(self(points[idx])), True)
        host = sums.reshape(-1).cpu()
        taken = len(batches) - (int(host[1]) if skip else 0)
        loss = _mean_over(float(host[0]), taken)
        if self.ae_loss == "emd":
            loss /= points.shape[1]
        res = {"loss": loss, "steps": len(batches)}
        if skip:
            res["skipped_steps"] = len(batches) - taken
        return res


# ----------------------------------------------------------------------------------------------------- training the samplers
class SamplerTrainStep:
    """The epoch of the SampleNet trainers around one of the steps above.  The optimiser holds the sampler's parameters, and with a
    reconstruction step built with fixed_ae=False (the auto-encoder trained together with the sampler) it may hold the auto-encoder's too;
    otherwise the steps freeze the task network.  Restated from:

        ClassificationStep / ProgressiveClassificationStep     classification/train_samplenet.py, train_samplenet_progressive.py
            step s (counted from 0, `self.step`): learning rate pointnet_learning_rate(s, batch_size, learning_rate, decay_step, decay_rate),
            and momentum 1 - pointnet_bn_decay(s, batch_size, decay_step) on the sampler's BatchNorm layers.  Defaults: lr 0.01, decay_step
            600000, decay_rate 0.7, batch_size 32.
        ReconstructionStep / ProgressiveReconstructionStep     reconstruction/sampler/train_samplenet.py, train_samplenet_progressive.py
            (samplenet_pointnet_ae.py:191-214): a constant learning rate (default 5e-4) or, with decay_steps (the configuration's
            exponential_decay), max(staircase_decay(learning_rate, epoch, decay_steps, 0.5), 1e-5) for epoch `self.epoch` counted from 0.
            The sampler's BatchNorm momentum is left as it is.  batch_size 50.  gauss_augment (None or {"mu", "sigma"}) and z_rotate
            augment every batch with ops.ae_augment before the step (general_utils.apply_augmentations; off by default, and then no launch
            is added).

    __call__(points (B, N, 3)[, labels (B,)]) is one step without a host synchronisation: the schedule, sampler.train(), zero_grad, the step's
    loss, backward, optimizer.step().  It returns the loss terms as detached device tensors: "loss" (the total) and the step's terms, and
    "correct" (the number of right predictions) where the step returns "pred".

    train_one_epoch(points (n, N, 3)[, labels (n,)]) runs an epoch over a device-resident set: a torch.randperm on the device, n // batch_size
    whole batches, every term summed in float64 on the device, one read-back.  in_out.PointCloudDataSet.next_batch (in_out.py:350-370)
    reshuffles when a batch would run past the end, so with int(n / batch_size) batches per epoch each epoch is a fresh permutation whose
    remainder is not used: the same epoch.  The classification scripts shuffle and drop the remainder per h5 file; here the set is one
    file.  Returns the means over batches of every term ("loss", ..., "steps"), with "accuracy" over the clouds seen where the step returns
    "pred".  For reconstruction it returns what _single_epoch_train returns (samplenet_pointnet_ae.py:291-353): with EMD loss_ae divided by
    the number of points, and "loss" recomposed as loss_ae + alpha * loss_simplification + lmbda * loss_projection.

    graphed=True runs every step as ONE CUDA-graph replay instead of the step's few dozen launches from Python, with the same results bit for
    bit (parameters, buffers, optimiser state, returned values).  The graph holds the schedule writes, the augmentation, the step and the
    addition of its terms into a float64 accumulator; the epoch's permutation, the per-step index_select into the static input buffers and
    the one read-back stay outside.  __call__ returns the same dict, of static buffers that the next step overwrites.  Captured launches
    freeze the learning rate and the BatchNorm momentum, so when either differs from the captured value (a staircase boundary of the
    schedule) the step is captured again and the old graph freed.  The optimiser must be one of graphs.ZERO_INIT_OPTIMIZERS (Adam, AdamW,
    Adamax, RAdam, RMSprop, Adadelta), whose warm-up the capture can undo, with capturable=True (else ValueError at construction), and the
    runner holds one input shape, dtype and device: another raises ValueError.  A graphed runner keeps a private memory pool and the
    static buffers for its lifetime.

    skip_nonfinite=True skips a step that goes non-finite: when a loss term the step returns, a gradient of a parameter the optimiser holds,
    or a parameter or floating buffer of the sampler after the update holds a NaN or an Inf, the step leaves every parameter, buffer
    (BatchNorm running statistics, num_batches_tracked) and optimiser state tensor exactly as it was before it.  The check and the restore
    run on the device with no read-back, eager or graphed.  With fixed_ae=False the auto-encoder's parameters and buffers are snapshot and
    restored with the sampler's.  __call__ adds "skipped" (0/1 int32 device tensor) to its dict; train_one_epoch
    leaves a skipped step's terms out of its sums, adds "skipped_steps" and takes its means over the steps taken (NaN if none was).  The
    schedule counters advance for a skipped batch all the same: it was consumed.  It needs an optimiser that graphed=True accepts (else
    ValueError), whose fresh state is zeros: optimiser state a skipped first step created comes back as zeros."""

    def __init__(self, step, optimizer, batch_size=None, learning_rate=None, decay_step=None, decay_rate=None, decay_steps=None,
                 gauss_augment=None, z_rotate=False, graphed=False, skip_nonfinite=False):
        self.classification = isinstance(step, ClassificationStep)
        if not self.classification and not isinstance(step, (ReconstructionStep, ProgressiveReconstructionStep)):
            raise TypeError("SamplerTrainStep wraps a ClassificationStep, ProgressiveClassificationStep, ReconstructionStep or "
                            "ProgressiveReconstructionStep, got %s" % type(step).__name__)
        if self.classification and (decay_steps is not None or gauss_augment is not None or z_rotate):
            raise ValueError("decay_steps, gauss_augment and z_rotate belong to the reconstruction trainers")
        if not self.classification and (decay_step is not None or decay_rate is not None):
            raise ValueError("decay_step and decay_rate belong to the classification trainers (reconstruction: decay_steps)")
        _check_augment(gauss_augment)
        self.task, self.optimizer = step, optimizer
        self.batch_size = int(batch_size if batch_size is not None else 32 if self.classification else 50)
        self.base_lr = float(learning_rate if learning_rate is not None else 0.01 if self.classification else 5e-4)
        self.decay_step = 600000 if decay_step is None else decay_step
        self.decay_rate = 0.7 if decay_rate is None else decay_rate
        self.decay_steps = decay_steps
        self.gauss_augment, self.z_rotate = gauss_augment, bool(z_rotate)
        self.step = 0
        self.epoch = 0
        self.graphed = bool(graphed)
        self._graph = None
        self.joint_ae = not self.classification and not step.fixed_ae
        trained = [step.sampler] + ([step.ae] if self.joint_ae else [])
        self._skip = _SkipNonfinite(trained, optimizer, type(self).__name__ + "(skip_nonfinite=True)") if skip_nonfinite else None
        if self.graphed:
            from .graphs import check_capturable

            check_capturable(optimizer, type(self).__name__ + "(graphed=True)")
            modules = [step.sampler, step.classifier if self.classification else step.ae]
            self._graph = _StepGraph(self, self._graph_step, modules, optimizer, ("step", "epoch"), self._skip is not None)

    def learning_rate(self):
        """The learning rate of the next step."""
        if self.classification:
            return pointnet_learning_rate(self.step, self.batch_size, self.base_lr, self.decay_step, self.decay_rate)
        if self.decay_steps is None:
            return self.base_lr
        return max(staircase_decay(self.base_lr, self.epoch, self.decay_steps, 0.5), 1e-5)

    def bn_momentum(self):
        """The sampler's BatchNorm momentum for the next step; None (left as it is) for reconstruction."""
        return 1.0 - pointnet_bn_decay(self.step, self.batch_size, self.decay_step) if self.classification else None

    def _schedule(self):
        """Set the schedule of the next step; returns its (learning rate, BatchNorm momentum)."""
        lr, momentum = self.learning_rate(), self.bn_momentum()
        _set_schedule(self.optimizer, lr, self.task.sampler, momentum)
        return lr, momentum

    def _step(self, points, labels=None):
        """One step without the step count: the dict __call__ returns."""
        sampler = self.task.sampler
        self._schedule()
        if self._skip is not None:
            self._skip.begin()
        points = _augment(points, self.gauss_augment, self.z_rotate)
        sampler.train()
        if self.joint_ae:
            self.task.ae.train()
        self.optimizer.zero_grad()
        total, terms = self.task.loss(points, labels) if self.classification else self.task.loss(points)
        total.backward()
        self.optimizer.step()
        out = {"loss": total.detach()}
        for k, v in terms.items():
            if k == "pred":
                out["correct"] = (v.detach().argmax(dim=1) == labels.long()).sum()
            else:
                out[k] = v.detach()
        if self._skip is not None:
            out["skipped"] = self._skip.end(list(out.values()))
        return out

    def _graph_step(self, points, labels=None):
        out = self._step(points, labels)
        return out, list(out.values())

    def __call__(self, points, labels=None):
        if self.classification and labels is None:
            raise ValueError("the classification step needs labels")
        if self.graphed:
            self._graph.bind(*((points, labels) if self.classification else (points,)))
            out = self._graph.replay(self._schedule())
        else:
            out = self._step(points, labels)
        self.step += 1
        return out

    def train_one_epoch(self, points, labels=None):
        if self.classification and labels is None:
            raise ValueError("the classification epoch needs labels")
        batches = _epoch_batches(points, self.batch_size)
        labels = None if labels is None else labels.to(points.device).reshape(-1)
        if self.graphed:
            sources = (points, labels) if self.classification else (points,)
            for s, idx in enumerate(batches):
                self._graph.select(sources, idx)
                keys = list(self._graph.replay(self._schedule(), first_of_epoch=s == 0))
                self.step += 1
            sums = self._graph.acc
        else:
            sums, keys = None, None
            for idx in batches:
                r = self(points[idx], None if labels is None else labels[idx])
                keys = list(r)
                v = _step_sums(list(r.values()), self._skip is not None)
                sums = v if sums is None else sums + v
        host = dict(zip(keys, sums.cpu().tolist()))
        steps = len(batches)
        taken = steps - int(host.pop("skipped", 0))
        self.epoch += 1
        res = {k: _mean_over(v, taken) for k, v in host.items() if k != "correct"}
        if "correct" in host:
            res["accuracy"] = _mean_over(host["correct"], taken * self.batch_size)
        if not self.classification:
            if getattr(self.task, "ae_loss", "chamfer") == "emd":
                res["loss_ae"] /= points.shape[1]
            res["loss"] = res["loss_ae"] + self.task.alpha * res["loss_simplification"] + self.task.lmbda * res["loss_projection"]
        res["steps"] = steps
        if self._skip is not None:
            res["skipped_steps"] = steps - taken
        return res
