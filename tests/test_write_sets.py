"""Write sets of the C-ABI entry points: every call writes the buffers it is given and nothing else.

Value tests cannot see a write that lands outside an entry's buffers: the memory it corrupts belongs to somebody else, and whether that
is memory a test reads depends on the caching allocator.  Here every buffer of a call -- inputs, layer parameters, BatchNorm buffers,
outputs, saved activations, workspaces, gradients -- is carved out of ONE device arena filled with a poison pattern, with a guard gap
between buffers, and the C ABI is called directly (the ops wrappers allocate internally).  Workspaces are carved at exactly their
*_workspace_bytes size, so an overrun of the declared size lands in a guard.  Around each call the arena is snapshotted and, after a
synchronise, checked for:
  * every word outside the call's declared write set bit-identical to the snapshot (inputs, weights, the forward workspace a backward
    reads, and every buffer of the calls before it);
  * every element the entry fully writes (outputs, all b*n rows of each saved activation, gradients) no longer holding the poison;
  * ticket / barrier words back to zero where the entry promises that.
A failure names the overwritten range, the buffer it lies in or follows (and how far past that buffer's end), and the first values
written there.  Sequences put three calls' buffers at different offsets of the same arena, so a write through a pointer kept from an
earlier call, or into an earlier call's saved activations, shows up as a write outside the current call's set.  A sequence is
deterministic: the layout does not depend on the allocator.

Generator cases cover the persistent conv-stack kernel's partition (snb200_debug_conv_stack_partition says which branch a shape
reaches on the device at hand): one slice per CTA at 64, 96 and 128 points, several slices per CTA at 96 and 128, a partial last slice, a
slice touching 8 clouds and clouds smaller than a thread's points."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

POISON = 0x7FA5A5A5      # a NaN bit pattern no kernel produces from finite inputs
GUARD = 4096             # bytes between two buffers of the arena
ALIGN = 256              # buffer alignment (one case uses ALIGN + 16: the least the conv stack accepts)
ARENA_BYTES = 1536 << 20
M = 32                   # sampled points of the generator tables: the last FC layer has 3 M outputs


# ------------------------------------------------------------------------------------------------------------------ the arena
def _addr(t):
    """Device address of a buffer, also of an empty one (whose data_ptr() is 0): what a 0-byte workspace is passed as."""
    return t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


class Region:
    def __init__(self, name, start, nbytes):
        self.name, self.start, self.nbytes = name, start, nbytes

    @property
    def end(self):
        return self.start + self.nbytes


class Arena:
    """One poisoned device buffer; carve() hands out views of it, GUARD bytes apart."""

    def __init__(self, nbytes=ARENA_BYTES, device="cuda"):
        self.words = torch.full((nbytes // 4,), POISON, dtype=torch.int32, device=device)
        self.bytes = self.words.view(torch.uint8)
        self.off = GUARD
        self.regions = []

    def carve(self, name, shape, dtype=torch.float32, skew=0, fill=None):
        shape = tuple(shape) if isinstance(shape, (tuple, list)) else (shape,)
        numel = 1
        for s in shape:
            numel *= s
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        start = (self.off + ALIGN - 1) // ALIGN * ALIGN + skew
        if start + nbytes + GUARD > self.bytes.numel():
            raise MemoryError("arena too small for %s (%d bytes at %d)" % (name, nbytes, start))
        self.off = start + nbytes + GUARD
        self.regions.append(Region(name, start, nbytes))
        t = self.bytes[start:start + max(nbytes, 16)].view(dtype)[:numel].view(shape)   # (a 0-byte buffer still has its own address)
        if fill is not None:
            t.copy_(fill)
        return t

    def region_of(self, t):
        start = _addr(t) - self.bytes.data_ptr()
        for r in self.regions:
            if r.start == start:
                return r
        raise KeyError("tensor is not a buffer of this arena")

    def locate(self, byte):
        """(description of where `byte` lies): inside a buffer, or past the end of the nearest buffer before it."""
        before = None
        for r in self.regions:
            if r.start <= byte < r.end:
                return "inside %s at byte %d of %d" % (r.name, byte - r.start, r.nbytes)
            if r.end <= byte and (before is None or r.end > before.end):
                before = r
        if before is None:
            return "in the arena's leading guard"
        return "%d bytes past the end of %s (%d bytes)" % (byte - before.end, before.name, before.nbytes)


def _word_mask(arena, tensors):
    mask = torch.zeros(arena.words.numel(), dtype=torch.bool, device=arena.words.device)
    for t in tensors:
        r = arena.region_of(t)
        mask[r.start // 4:(r.end + 3) // 4] = True
    return mask


def _describe(arena, stray, snap, limit=8):
    idx = stray.nonzero().flatten().cpu().tolist()
    runs, s0, prev = [], idx[0], idx[0]
    for i in idx[1:]:
        if i != prev + 1:
            runs.append((s0, prev))
            s0 = i
        prev = i
    runs.append((s0, prev))
    lines = ["%d words written outside the write set, in %d ranges:" % (len(idx), len(runs))]
    for a, b in runs[:limit]:
        vals = arena.words[a:min(b + 1, a + 4)]
        old = snap[a:min(b + 1, a + 4)]
        lines.append("  bytes [%d, %d): %s; first words %s = %s (were %s)" % (
            4 * a, 4 * (b + 1), arena.locate(4 * a), ["0x%08x" % (v & 0xFFFFFFFF) for v in vals.tolist()],
            ["%.6g" % v for v in vals.view(torch.float32).tolist()], ["0x%08x" % (v & 0xFFFFFFFF) for v in old.tolist()]))
    if len(runs) > limit:
        lines.append("  ... %d more ranges" % (len(runs) - limit))
    return lines


def run_checked(arena, label, call, writes=(), full=(), zero=()):
    """Runs call() between two snapshots of the arena.  writes: buffers the call may write; full: buffers (also in its write set) whose
    every element it must write; zero: (buffer, what) pairs that must hold zero afterwards.  Returns the list of findings (empty = clean)."""
    torch.cuda.synchronize()
    snap = arena.words.clone()
    call()
    torch.cuda.synchronize()
    stray = (arena.words != snap) & ~_word_mask(arena, list(writes) + list(full))
    report = []
    if bool(stray.any()):
        report += _describe(arena, stray, snap)
    for t in full:
        r = arena.region_of(t)
        left = int((arena.words[r.start // 4:r.end // 4] == POISON).sum())
        if left:
            report.append("%s: %d of %d words never written" % (r.name, left, r.nbytes // 4))
    for t, what in zero:
        if bool((t != 0).any()):
            report.append("%s not back to zero: %s" % (what, t.flatten()[:8].tolist()))
    return ["%s: %s" % (label, line) for line in report]


def assert_clean(report):
    assert not report, "\n".join(report)


@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


@pytest.fixture(scope="module")
def arena_store(sb):
    return {}


@pytest.fixture
def arena(arena_store):
    """The module's arena, re-poisoned and empty for every test."""
    a = arena_store.get("a")
    if a is None:
        a = arena_store["a"] = Arena()
    a.words.fill_(POISON)
    a.off, a.regions = GUARD, []
    return a


# ------------------------------------------------------------------------------------------------------------------ harness self-test
@pytest.mark.gpu
def test_harness_reports_a_write_past_a_buffer_and_into_an_earlier_call(sb, arena):
    x1 = arena.carve("call1.out", (100,), fill=torch.zeros(100))
    x2 = arena.carve("call2.out", (37,), fill=torch.zeros(37))
    past = arena.bytes[arena.region_of(x2).end:].view(torch.float32)
    rep = run_checked(arena, "past the end", lambda: (x2.fill_(1.0), past[0].fill_(2.0)), writes=[x2], full=[x2])
    assert len(rep) == 2 and "0 bytes past the end of call2.out" in rep[1] and "0x40000000" in rep[1], rep
    rep = run_checked(arena, "earlier call", lambda: (x2.fill_(1.0), x1[17].fill_(3.0)), writes=[x2], full=[x2])
    assert len(rep) == 2 and "inside call1.out at byte 68 of 400" in rep[1], rep
    x3 = arena.carve("call3.out", (37,))
    rep = run_checked(arena, "unwritten", lambda: x3[:-1].fill_(1.0), writes=[x3], full=[x3])
    assert rep == ["unwritten: call3.out: 1 of 37 words never written"], rep
    ticket = arena.carve("ticket", (1,), dtype=torch.int32, fill=torch.zeros(1, dtype=torch.int32))
    rep = run_checked(arena, "ticket", lambda: ticket.fill_(5), writes=[ticket], zero=[(ticket, "ticket")])
    assert len(rep) == 1 and "ticket not back to zero" in rep[0], rep
    assert run_checked(arena, "clean", lambda: x2.fill_(4.0), writes=[x2], full=[x2]) == []


# ------------------------------------------------------------------------------------------------------------------ generator
# conv widths, FC widths, FC BatchNorm, FC ReLU, eps, backward (the fused CUDA backward takes the table)
TABLES = {
    "reg": ([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3 * M], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5, True),
    "cls": ([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3 * M], [1, 1, 1, 1], [1, 1, 1, 0], 1e-3, False),
    "k128": ([3, 128, 128, 128], [128, 256, 3 * M], [1, 0], [1, 0], 1e-5, True),
    "k32": ([3, 32, 32, 128, 72], [72, 64, 3 * M], [1, 0], [1, 0], 1e-5, False),
    # a 42-wide last conv layer (c_in & 3 = 2 for fc1: scalar row and weight staging); then every FC input unaligned as well
    "narrow42": ([3, 64, 64, 64, 128, 42], [42, 256, 256, 256, 3 * M], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5, False),
    "unaligned": ([3, 64, 64, 64, 128, 42], [42, 50, 30, 99], [1, 1, 0], [1, 1, 0], 1e-5, False),
}


def _partition(sb, b, n):
    v = [ctypes.c_int() for _ in range(5)]
    sb._lib.check(sb._lib.lib().snb200_debug_conv_stack_partition(b, n, *[ctypes.byref(t) for t in v]), "debug_conv_stack_partition")
    ppc, slices, grid, per_cta, slots = (t.value for t in v)
    total = b * n
    clouds = max((min(total, (s + 1) * ppc) - 1) // n - (s * ppc) // n + 1 for s in range(slices))
    return dict(ppc=ppc, slices=slices, grid=grid, per_cta=per_cta, slots=slots, multi=per_cta > 1, partial=total % ppc != 0,
                clouds=clouds, n_below_thread=n < ppc // 4)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _branch_shape(kind, ppc):
    """(b, n = 1000) that reaches the given partition branch on this device: one slice per CTA holds the batch at up to sms * ppc points,
    two rounds of slices at up to 2 * sms * ppc."""
    lo = {("single", 96): 64, ("single", 128): 96, ("multi", 96): 128, ("multi", 128): 192}[(kind, ppc)]
    return _sms() * (lo + 16) // 1000, 1000


def make_table(arena, tag, name, seed, skew=0):
    """(conv specs, fc specs) of a layer table with every tensor carved from the arena."""
    conv_w, fc_w, fc_bn, fc_relu, eps, _ = TABLES[name]
    g = torch.Generator().manual_seed(seed)

    def layer(kind, i, c_in, c_out, bn, relu):
        nm = "%s.%s%d" % (tag, kind, i)
        w = arena.carve(nm + ".weight", (c_out, c_in), skew=skew, fill=(torch.randn(c_out, c_in, generator=g) / c_in ** 0.5))
        b = arena.carve(nm + ".bias", (c_out,), fill=0.1 * torch.randn(c_out, generator=g))
        spec = dict(weight=w, bias=b, relu=bool(relu), bn=None)
        if bn:
            spec["bn"] = (arena.carve(nm + ".bn_weight", (c_out,), fill=1 + 0.2 * torch.randn(c_out, generator=g)),
                          arena.carve(nm + ".bn_bias", (c_out,), fill=0.1 * torch.randn(c_out, generator=g)),
                          arena.carve(nm + ".running_mean", (c_out,), fill=0.2 * torch.randn(c_out, generator=g)),
                          arena.carve(nm + ".running_var", (c_out,), fill=0.5 + torch.rand(c_out, generator=g)),
                          eps, 0.1,
                          arena.carve(nm + ".num_batches_tracked", (1,), dtype=torch.int64, fill=torch.zeros(1, dtype=torch.int64)))
        return spec

    conv = [layer("conv", i, conv_w[i], conv_w[i + 1], True, True) for i in range(len(conv_w) - 1)]
    fc = [layer("fc", i, fc_w[i], fc_w[i + 1], fc_bn[i], fc_relu[i]) for i in range(len(fc_w) - 1)]
    return conv, fc


def _bn_buffers(specs):
    return [t for s in specs if s["bn"] is not None for t in (s["bn"][2], s["bn"][3], s["bn"][6])]


class GenCall:
    """One generator call's buffers, all carved from the arena: input, layer tables, outputs, saved activations, workspaces and gradients."""

    def __init__(self, sb, arena, tag, name, b, n, layout, inner, seed=0, skew=0, ws=None):
        self.sb, self.arena, self.tag = sb, arena, tag
        self.b, self.n, self.layout, self.inner = b, n, layout, inner
        self.lay = sb._lib.BNC if layout == "bnc" else sb._lib.BCN
        x = torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed + 7)) - 0.5
        self.x = arena.carve(tag + ".x", (b, n, 3) if layout == "bnc" else (b, 3, n), skew=skew,
                             fill=x if layout == "bnc" else x.permute(0, 2, 1))
        self.conv_specs, self.fc_specs = make_table(arena, tag, name, seed, skew=skew)
        self.conv, _ = sb.ops.make_layers(self.conv_specs)
        self.fc, _ = sb.ops.make_layers(self.fc_specs)
        for arr, specs in ((self.conv, self.conv_specs), (self.fc, self.fc_specs)):   # the tables point into the arena, no copies
            assert all(arr[i].weight == s["weight"].data_ptr() and arr[i].bias == s["bias"].data_ptr() for i, s in enumerate(specs))
        self.nc, self.nf = len(self.conv_specs), len(self.fc_specs)
        lib = sb._lib.lib()
        self.wsb = int(lib.snb200_generator_workspace_bytes(b, n, self.nc, self.conv, self.nf, self.fc))
        # (the skew applies to the caller's tensors -- the 16-byte minimum the ABI states; workspaces keep the allocator's alignment)
        self.ws = ws if ws is not None else arena.carve(tag + ".workspace", (self.wsb,), dtype=torch.uint8)
        self.out = arena.carve(tag + ".out", (b, self.fc[self.nf - 1].c_out), skew=skew)
        self.feat = arena.carve(tag + ".feat", (b, self.conv[self.nc - 1].c_out), skew=skew)
        self.zs = []

    def bn_buffers(self):
        return _bn_buffers(self.conv_specs + self.fc_specs)

    def forward(self, training, flags=0):
        lib = self.sb._lib.lib()
        rc = [0]

        def call():
            rc[0] = lib.snb200_generator_forward(self.b, self.n, self.lay, self.x.data_ptr(), self.nc, self.conv, self.nf, self.fc, int(training),
                                                 self.out.data_ptr(), self.inner, self.feat.data_ptr(), flags, _addr(self.ws), self.wsb, None)
        writes = [self.ws] + (self.bn_buffers() if training else [])
        rep = run_checked(self.arena, "%s generator_forward(training=%d, flags=%d)" % (self.tag, training, flags), call, writes,
                          full=[self.out, self.feat], zero=self._primed_words(flags))
        self.sb._lib.check(rc[0], "generator_forward")
        return rep

    def _primed_words(self, flags):
        if not flags & self.sb._lib.GEN_WORKSPACE_PRIMED:
            return []
        return [(self.ws[:256], "moments, grid-barrier and exit words of the PRIMED workspace")]

    def train_forward(self, layers=False, flags=0):
        lib = self.sb._lib.lib()
        entry = "generator_layers_train_forward" if layers else "generator_train_forward"
        self.zs = [self.arena.carve("%s.zsave[%d]" % (self.tag, l), (self.b * self.n, self.conv[l].c_out)) for l in range(self.nc)]
        zp = (ctypes.c_void_p * self.nc)(*[z.data_ptr() for z in self.zs])
        rc = [0]

        def call():
            rc[0] = getattr(lib, "snb200_" + entry)(self.b, self.n, self.lay, self.x.data_ptr(), self.nc, self.conv, self.nf, self.fc,
                                                     self.out.data_ptr(), self.inner, self.feat.data_ptr(), zp, flags, _addr(self.ws),
                                                     self.wsb, None)
        rep = run_checked(self.arena, "%s %s" % (self.tag, entry), call, [self.ws] + self.bn_buffers(), full=[self.out, self.feat] + self.zs,
                          zero=self._primed_words(flags))
        self.sb._lib.check(rc[0], entry)
        return rep

    def backward(self, layers=False):
        sb, lib, arena = self.sb, self.sb._lib.lib(), self.arena
        entry = "generator_layers_backward" if layers else "generator_backward"
        bwsb = int(getattr(lib, "snb200_%s_workspace_bytes" % entry)(self.b, self.n, self.nc, self.conv, self.nf, self.fc))
        bws = arena.carve(self.tag + ".backward_workspace", (bwsb,), dtype=torch.uint8)
        grad_out = arena.carve(self.tag + ".grad_out", tuple(self.out.shape), fill=torch.randn(tuple(self.out.shape),
                                                                                            generator=torch.Generator().manual_seed(3)))
        grads = []

        def gstructs(specs, kind):
            arr = (sb._lib.LayerGrad * len(specs))()
            for i, s in enumerate(specs):
                c_out, c_in = s["weight"].shape
                nm = "%s.grad.%s%d" % (self.tag, kind, i)
                g = [arena.carve(nm + ".weight", (c_out, c_in)), arena.carve(nm + ".bias", (c_out,))]
                if s["bn"] is not None:
                    g += [arena.carve(nm + ".bn_weight", (c_out,)), arena.carve(nm + ".bn_bias", (c_out,))]
                arr[i].weight, arr[i].bias = g[0].data_ptr(), g[1].data_ptr()
                arr[i].bn_weight, arr[i].bn_bias = (g[2].data_ptr(), g[3].data_ptr()) if len(g) > 2 else (None, None)
                grads.extend(g)
            return arr
        gconv, gfc = gstructs(self.conv_specs, "conv"), gstructs(self.fc_specs, "fc")
        zp = (ctypes.c_void_p * self.nc)(*[z.data_ptr() for z in self.zs])
        rc = [0]

        def call():
            rc[0] = getattr(lib, "snb200_" + entry)(self.b, self.n, self.lay, self.x.data_ptr(), self.nc, self.conv, self.nf, self.fc, zp,
                                                     _addr(self.ws), grad_out.data_ptr(), self.inner, gconv, gfc, _addr(bws), bwsb, None)
        rep = run_checked(arena, "%s %s" % (self.tag, entry), call, [bws], full=grads)
        sb._lib.check(rc[0], entry)
        return rep


# (table, b, n, layout, out_transpose_inner, expected branch).  Branch keys: multi (several slices per CTA), ppc, partial (last slice
# partial), clouds (most clouds one slice touches), n_below_thread (a cloud is shorter than a thread's points).  The named shapes are
# those of the saved-activation failures of the fused training path, registration at batch 1, and a small evaluation batch.
GEN_SHAPES = [
    pytest.param("reg", 7, 1000, "bnc", M, dict(multi=False, ppc=64, partial=True), id="reg-7x1000-bnc-inner"),
    pytest.param("reg", 16, 333, "bcn", 0, dict(multi=False, ppc=64), id="reg-16x333-bcn"),
    pytest.param("reg", 7, 333, "bnc", 0, dict(multi=False, ppc=64), id="reg-7x333"),
    pytest.param("reg", 4, 256, "bnc", 0, dict(multi=False, ppc=64, partial=False), id="reg-4x256"),
    pytest.param("reg", 64, 10, "bnc", 0, dict(multi=False, ppc=64, clouds=8, n_below_thread=True), id="reg-64x10-8clouds"),
    pytest.param("k128", ("single", 96), None, "bnc", 0, dict(multi=False, ppc=96), id="k128-single96"),
    pytest.param("reg", ("single", 128), None, "bcn", 0, dict(multi=False, ppc=128), id="reg-single128-bcn"),
    pytest.param("reg", ("multi", 96), None, "bnc", M, dict(multi=True, ppc=96), id="reg-multi96-inner"),
    pytest.param("k128", ("multi", 128), None, "bnc", 0, dict(multi=True, ppc=128), id="k128-multi128"),
]


def _shape(b, n):
    return _branch_shape(*b) if isinstance(b, tuple) else (b, n)


def _check_branch(sb, b, n, expect):
    part = _partition(sb, b, n)
    got = {k: part[k] for k in expect}
    assert got == expect, ("partition of %d x %d on %d SMs" % (b, n, _sms()), part)
    return part


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,inner,expect", GEN_SHAPES)
def test_generator_training_sequence_writes_only_its_buffers(sb, arena, table, b, n, layout, inner, expect):
    """Three fused training steps (train_forward + backward) in a row, each on its own buffers: neither entry writes outside its set, and
    nothing touches an earlier step's saved activations."""
    b, n = _shape(b, n)
    _check_branch(sb, b, n, expect)
    if not TABLES[table][5]:
        pytest.skip("the fused backward does not take this table")
    rep = []
    for i in range(3):
        c = GenCall(sb, arena, "step%d" % i, table, b, n, layout, inner, seed=0)
        rep += c.train_forward()
        rep += c.backward()
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,inner,expect", GEN_SHAPES)
def test_generator_forward_modes_write_only_their_buffers(sb, arena, table, b, n, layout, inner, expect):
    """generator_forward in eval and training mode, with the fused head and with SNB200_GEN_SEPARATE_HEAD, each call on its own buffers."""
    b, n = _shape(b, n)
    _check_branch(sb, b, n, expect)
    rep = []
    for i, (training, flags) in enumerate([(0, 0), (1, 0), (0, sb._lib.GEN_SEPARATE_HEAD), (1, sb._lib.GEN_SEPARATE_HEAD)]):
        rep += GenCall(sb, arena, "call%d" % i, table, b, n, layout, inner, seed=1).forward(training, flags)
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,inner,expect", GEN_SHAPES)
def test_generator_primed_sequence_writes_only_its_buffers(sb, arena, table, b, n, layout, inner, expect):
    """Three SNB200_GEN_WORKSPACE_PRIMED training forwards on ONE workspace (the other buffers at new offsets every call): the kernel
    cleans its own scratch and leaves the moments, barrier and exit words zero for the next call."""
    b, n = _shape(b, n)
    _check_branch(sb, b, n, expect)
    first = GenCall(sb, arena, "call0", table, b, n, layout, inner, seed=2)
    first.ws.zero_()
    rep = first.forward(1, sb._lib.GEN_WORKSPACE_PRIMED)
    for i in (1, 2):
        rep += GenCall(sb, arena, "call%d" % i, table, b, n, layout, inner, seed=2, ws=first.ws).forward(1, sb._lib.GEN_WORKSPACE_PRIMED)
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,inner,expect", [p for p in GEN_SHAPES if TABLES[p.values[0]][5]])
def test_generator_layers_route_writes_only_its_buffers(sb, arena, table, b, n, layout, inner, expect):
    """The per-layer training route at the same shapes (tensor-core layer kernels + cluster head, then the same backward kernels)."""
    b, n = _shape(b, n)
    rep = []
    for i in range(2):
        c = GenCall(sb, arena, "step%d" % i, table, b, n, layout, inner, seed=3)
        rep += c.train_forward(layers=True)
        rep += c.backward(layers=True)
    assert_clean(rep)


@pytest.mark.gpu
def test_generator_eval_at_batch_one_and_least_alignment(sb, arena):
    """Registration's evaluation call (one cloud of 1024 points: 16 CTAs) with every buffer 16 bytes off a 256-byte boundary."""
    assert _partition(sb, 1, 1024)["per_cta"] == 1
    rep = []
    for i, table in enumerate(["reg", "cls", "k32", "narrow42", "unaligned"]):
        rep += GenCall(sb, arena, "call%d" % i, table, 1, 1024, "bnc", 0, seed=4, skew=16).forward(0, 0)
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["cls", "k32", "k128", "narrow42", "unaligned"])
def test_generator_tables_write_only_their_buffers(sb, arena, table):
    """Every layer table the persistent kernel takes, at one slice per CTA and at several."""
    rep = []
    for i, (b, n) in enumerate([(7, 1000), _branch_shape("multi", 128)]):
        rep += GenCall(sb, arena, "call%d" % i, table, b, n, "bnc", 0, seed=5).forward(1, 0)
        rep += GenCall(sb, arena, "call%d.eval" % i, table, b, n, "bnc", 0, seed=5).forward(0, 0)
    assert_clean(rep)


def test_harness_layout_arithmetic():
    """The carving and locating logic on the CPU: offsets, guards, skew and the nearest-buffer report."""
    a = Arena(1 << 16, device="cpu")
    t1 = a.carve("one", (10,))
    t2 = a.carve("two", (3,), dtype=torch.int64, skew=16)
    r1, r2 = a.region_of(t1), a.region_of(t2)
    assert r1.start % ALIGN == 0 and r2.start % ALIGN == 16 and r2.start - r1.end >= GUARD
    assert a.locate(r1.end + 4) == "4 bytes past the end of one (40 bytes)"
    assert a.locate(r2.start + 8) == "inside two at byte 8 of 24"
    assert a.locate(0) == "in the arena's leading guard"
    with pytest.raises(MemoryError):
        a.carve("big", (1 << 16,))


# ------------------------------------------------------------------------------------------------------------------ recent entries
def _vp(t):
    return None if t is None else t.data_ptr()


def _ptrs(ts):
    return (ctypes.c_void_p * max(len(ts), 1))(*[t.data_ptr() for t in ts])


def _rand(g, *shape, scale=1.0, shift=0.0):
    return torch.rand(*shape, generator=g) * scale + shift


def make_fc_table(arena, tag, widths, relu, bn=False, seed=0):
    """A frozen FC / conv layer table carved from the arena (eval-mode BatchNorm with running statistics when bn)."""
    g = torch.Generator().manual_seed(seed)
    specs = []
    for i in range(len(widths) - 1):
        c_in, c_out = widths[i], widths[i + 1]
        nm = "%s.layer%d" % (tag, i)
        s = dict(weight=arena.carve(nm + ".weight", (c_out, c_in), fill=(torch.rand(c_out, c_in, generator=g) - 0.5) * 2 / c_in ** 0.5),
                 bias=arena.carve(nm + ".bias", (c_out,), fill=0.1 * (torch.rand(c_out, generator=g) - 0.5)), relu=bool(relu[i]), bn=None)
        if bn:
            s["bn"] = (arena.carve(nm + ".bn_weight", (c_out,), fill=_rand(g, c_out, shift=0.5)),
                       arena.carve(nm + ".bn_bias", (c_out,), fill=_rand(g, c_out, scale=0.2, shift=-0.1)),
                       arena.carve(nm + ".running_mean", (c_out,), fill=_rand(g, c_out, scale=0.2, shift=-0.1)),
                       arena.carve(nm + ".running_var", (c_out,), fill=_rand(g, c_out, shift=0.5)), 1e-3, 0.1)
        specs.append(s)
    return specs


# (widths, ReLU per layer, BatchNorm, rows, expected backward workspace: "none" = no split anywhere (the 256-byte placeholder), "split" =
# layer 0's output channels split over grid.y, whose partial blocks the sum launch adds into grad_in)
MLP_CASES = [
    pytest.param([4096, 256], [0], False, 16, "none", id="one-layer-4096-unsplit"),
    pytest.param([64, 1024], [0], False, 5, "split", id="one-layer-64-split8"),
    pytest.param([2048, 1024, 1024, 512, 512, 256, 7], [1, 1, 1, 1, 1, 0], False, 32, "split", id="pcrnet-b32"),
    pytest.param([2048, 1024, 1024, 512, 512, 256, 7], [1, 1, 1, 1, 1, 0], False, 1, "split", id="pcrnet-b1"),
    pytest.param([1024, 512, 256, 40], [1, 1, 0], True, 64, "split", id="bn-classifier-b64"),
    pytest.param([256, 9], [0], True, 3, "none", id="bn-one-layer-narrow"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("widths,relu,bn,b,branch", MLP_CASES)
def test_frozen_mlp_writes_only_its_buffers(sb, arena, widths, relu, bn, b, branch):
    lib, ops = sb._lib.lib(), sb.ops
    name = "frozen_mlp_bn" if bn else "frozen_mlp"
    entry = lambda what: getattr(lib, "snb200_%s_%s" % (name, what))
    specs = make_fc_table(arena, "mlp", widths, relu, bn)
    table, _ = ops.make_layers(specs)
    nl = len(specs)
    assert entry("supported")(b, nl, table)
    bwsb = int(entry("backward_workspace_bytes")(b, nl, table))
    assert (bwsb == 256) == (branch == "none"), (branch, bwsb)
    if branch == "split":   # layer 0's partial blocks lead the workspace: more than one of them
        assert bwsb >= 2 * b * widths[0] * 4 if nl == 1 else bwsb > 256
    g = torch.Generator().manual_seed(b)
    x = arena.carve("x", (b, widths[0]), fill=torch.rand(b, widths[0], generator=g) - 0.5)
    rep = []
    saves = []
    for keep in (1, 0):
        out = arena.carve("out.keep%d" % keep, (b, widths[-1]))
        asave = [arena.carve("asave%d.keep%d" % (l, keep), (b, widths[l + 1])) for l in range(nl - 1)] if keep else []
        wsb = int(entry("workspace_bytes")(b, nl, table, keep))
        ws = arena.carve("forward_workspace.keep%d" % keep, (wsb,), dtype=torch.uint8)
        rc = []
        rep += run_checked(arena, "%s_forward(with_save=%d)" % (name, keep), lambda: rc.append(entry("forward")(
            b, x.data_ptr(), nl, table, out.data_ptr(), _ptrs(asave) if keep else None, _addr(ws), wsb, None)), [ws], full=[out] + asave)
        sb._lib.check(rc[0], name + "_forward")
        saves.append(asave)
    for i in range(2):   # two backward calls on their own buffers, the second behind the first
        go = arena.carve("grad_out%d" % i, (b, widths[-1]), fill=torch.randn(b, widths[-1], generator=g))
        gin = arena.carve("grad_in%d" % i, (b, widths[0]))
        bws = arena.carve("backward_workspace%d" % i, (bwsb,), dtype=torch.uint8)
        rc = []
        rep += run_checked(arena, "%s_backward #%d" % (name, i), lambda: rc.append(entry("backward")(
            b, nl, table, _ptrs(saves[0]), go.data_ptr(), gin.data_ptr(), _addr(bws), bwsb, None)), [bws], full=[gin])
        sb._lib.check(rc[0], name + "_backward")
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,k,chunks", [(3, 128, 3, 1), (2, 1000, 64, 8), (5, 333, 17, 3), (1, 129, 64, 2)])
def test_point_transform_writes_only_its_buffers(sb, arena, b, n, k, chunks):
    """Forward, and the backward with one 128-point chunk per cloud (no workspace) and with several (per-chunk partial grad_T blocks)."""
    lib = sb._lib.lib()
    wsb = int(lib.snb200_point_transform_workspace_bytes(b, n, k))
    assert (wsb == 0) == (chunks == 1) and (n + 127) // 128 == chunks, wsb
    g = torch.Generator().manual_seed(n)
    x = arena.carve("x", (b, n, k), fill=torch.rand(b, n, k, generator=g) - 0.5)
    T = arena.carve("T", (b, k, k), fill=torch.rand(b, k, k, generator=g) - 0.5)
    out = arena.carve("out", (b, n, k))
    rc = []
    rep = run_checked(arena, "point_transform_forward", lambda: rc.append(lib.snb200_point_transform_forward(
        b, n, k, x.data_ptr(), T.data_ptr(), out.data_ptr(), None)), full=[out])
    for i in range(2):
        go = arena.carve("grad_out%d" % i, (b, n, k), fill=torch.randn(b, n, k, generator=g))
        gx, gT = arena.carve("grad_x%d" % i, (b, n, k)), arena.carve("grad_T%d" % i, (b, k, k))
        ws = arena.carve("workspace%d" % i, (wsb,), dtype=torch.uint8)
        rep += run_checked(arena, "point_transform_backward #%d" % i, lambda: rc.append(lib.snb200_point_transform_backward(
            b, n, k, x.data_ptr(), T.data_ptr(), go.data_ptr(), gx.data_ptr(), gT.data_ptr(), _addr(ws), wsb, None)), [ws], full=[gx, gT])
    assert rc == [0, 0, 0], sb._lib.lib().snb200_last_error()
    assert_clean(rep)


def _pose_inputs(arena, tag, b, m, g):
    q = torch.randn(b, 4, generator=g)
    y = torch.cat([q * 1.3, 0.1 * torch.randn(b, 3, generator=g)], 1)
    igt = torch.cat([q / q.norm(dim=1, keepdim=True), 0.1 * torch.randn(b, 3, generator=g)], 1)
    return (arena.carve(tag + ".y", (b, 7), fill=y), arena.carve(tag + ".p0", (b, m, 3), fill=torch.rand(b, m, 3, generator=g) - 0.5),
            arena.carve(tag + ".p1", (b, m, 3), fill=torch.rand(b, m, 3, generator=g) - 0.5), arena.carve(tag + ".igt", (b, 7), fill=igt))


@pytest.mark.gpu
@pytest.mark.parametrize("b,m", [(1, 64), (32, 64), (7, 1024)])
def test_pose_loss_writes_only_its_buffers_and_returns_the_ticket(sb, arena, b, m):
    """Forward (the last CTA adds the per-pair sums and puts the ticket back to zero) and backward, three pairs of calls in a row."""
    lib = sb._lib.lib()
    g = torch.Generator().manual_seed(b * m)
    wsb = int(lib.snb200_pose_loss_workspace_bytes(b, m))
    rep, rc = [], []
    for i in range(3):
        tag = "call%d" % i
        y, p0, p1, igt = _pose_inputs(arena, tag, b, m, g)
        twist, terms = arena.carve(tag + ".twist", (b, 7)), arena.carve(tag + ".terms", (5,))
        idx01 = arena.carve(tag + ".idx01", (b, m), dtype=torch.int32)
        idx10 = arena.carve(tag + ".idx10", (b, m), dtype=torch.int32)
        ws = arena.carve(tag + ".workspace", (wsb,), dtype=torch.uint8)
        ticket = arena.carve(tag + ".ticket", (1,), dtype=torch.int32, fill=torch.zeros(1, dtype=torch.int32))
        rep += run_checked(arena, tag + " pose_loss_forward", lambda: rc.append(lib.snb200_pose_loss_forward(
            b, m, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), twist.data_ptr(), idx01.data_ptr(), idx10.data_ptr(),
            terms.data_ptr(), _addr(ws), wsb, ticket.data_ptr(), None)), [ws, ticket], full=[twist, idx01, idx10, terms],
            zero=[(ticket, tag + " ticket")])
        gt = arena.carve(tag + ".grad_terms", (5,), fill=torch.tensor([1.0, 0.5, 0.25, 3.0, 2.0]))
        gy, g0, g1 = arena.carve(tag + ".grad_y", (b, 7)), arena.carve(tag + ".grad_p0", (b, m, 3)), arena.carve(tag + ".grad_p1", (b, m, 3))
        rep += run_checked(arena, tag + " pose_loss_backward", lambda: rc.append(lib.snb200_pose_loss_backward(
            b, m, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), idx01.data_ptr(), idx10.data_ptr(), gt.data_ptr(), gy.data_ptr(),
            g0.data_ptr(), g1.data_ptr(), None)), full=[gy, g0, g1])
    assert rc == [0] * 6, lib.snb200_last_error()
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("b,m,ms", [(1, 1024, 0), (32, 64, 0), (32, 256, 64), (5, 100, 100)])
def test_pose_eval_writes_only_its_buffers(sb, arena, b, m, ms):
    """With the sampled pair (p0s, p1s: the consistency column) and without it (column 0)."""
    lib = sb._lib.lib()
    g = torch.Generator().manual_seed(b + m)
    y, p0, p1, igt = _pose_inputs(arena, "in", b, m, g)
    p0s = arena.carve("p0s", (b, ms, 3), fill=torch.rand(b, ms, 3, generator=g) - 0.5) if ms else None
    p1s = arena.carve("p1s", (b, ms, 3), fill=torch.rand(b, ms, 3, generator=g) - 0.5) if ms else None
    per_pair, twist = arena.carve("per_pair", (b, 6)), arena.carve("twist", (b, 7))
    rc = []
    rep = run_checked(arena, "pose_eval(ms=%d)" % ms, lambda: rc.append(lib.snb200_pose_eval(
        b, m, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), ms, _vp(p0s), _vp(p1s), per_pair.data_ptr(), twist.data_ptr(), None)),
        full=[per_pair, twist])
    assert rc == [0], lib.snb200_last_error()
    assert_clean(rep)
    if not ms:
        assert bool((per_pair[:, 5] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("b,b2,n,m", [(6, 2, 300, 200), (8, 1, 64, 2048), (3, 3, 1000, 17), (16, 4, 2048, 64)])
def test_chamfer_per_cloud_writes_only_its_buffers(sb, arena, b, b2, n, m):
    """Per-CTA partials in the workspace, added in tile order; xyz2 holds b2 <= b clouds."""
    lib = sb._lib.lib()
    g = torch.Generator().manual_seed(n + m)
    wsb = int(lib.snb200_chamfer_per_cloud_workspace_bytes(b, n, m))
    rep, rc = [], []
    for i in range(2):
        x1 = arena.carve("call%d.xyz1" % i, (b, n, 3), fill=torch.rand(b, n, 3, generator=g))
        x2 = arena.carve("call%d.xyz2" % i, (b2, m, 3), fill=torch.rand(b2, m, 3, generator=g))
        sums, ws = arena.carve("call%d.sums" % i, (b, 2)), arena.carve("call%d.workspace" % i, (wsb,), dtype=torch.uint8)
        rep += run_checked(arena, "chamfer_per_cloud #%d" % i, lambda: rc.append(lib.snb200_chamfer_per_cloud(
            b, n, x1.data_ptr(), m, x2.data_ptr(), b2, sums.data_ptr(), _addr(ws), wsb, None)), [ws], full=[sums])
    assert rc == [0, 0], lib.snb200_last_error()
    assert_clean(rep)


# (conv widths, act_input, tap, b, n, prefix sizes)
ENC_CASES = [
    pytest.param([3, 64, 64, 64, 128, 1024], 0, 1, 4, 300, [8, 100, 300], id="cloud-tap1"),
    pytest.param([3, 64, 64, 64, 128, 1024], 0, -1, 1, 1024, [1024], id="cloud-notap-b1"),
    pytest.param([64, 64, 128, 1024], 1, -1, 5, 333, [1, 7, 128, 333], id="act-input"),
    pytest.param([64, 64, 128, 256], 1, 0, 32, 128, [32, 64, 128], id="act-input-tap0"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("widths,act,tap,b,n,sizes", ENC_CASES)
def test_frozen_encoder_ex_writes_only_its_buffers(sb, arena, widths, act, tap, b, n, sizes):
    """Forward with saved activations (and a tapped hidden activation), then the backward with and without the tap's gradient."""
    lib, ops = sb._lib.lib(), sb.ops
    specs = make_fc_table(arena, "enc", widths, [1] * (len(widths) - 2) + [1], bn=True, seed=b)
    conv, _ = ops.make_layers(specs)
    nconv, npf = len(specs), len(sizes)
    assert lib.snb200_frozen_encoder_ex_supported(b, n, act, nconv, conv, npf, tap)
    csz = (ctypes.c_int * npf)(*sizes)
    g = torch.Generator().manual_seed(n)
    c_in = widths[0]
    x = arena.carve("in", (b, n, c_in), fill=torch.rand(b, n, c_in, generator=g) - (0.5 if not act else 0.0))
    C = widths[-1]
    pooled, route = arena.carve("pooled", (npf, b, C)), arena.carve("route", (npf, b, C), dtype=torch.int32)
    tap_out = arena.carve("tap_out", (b * n, widths[tap + 1])) if tap >= 0 else None
    zs = [arena.carve("zsave[%d]" % l, (b * n, widths[l + 1])) for l in range(nconv - 1)]
    wsb = int(lib.snb200_frozen_encoder_ex_workspace_bytes(b, n, act, nconv, conv, npf, tap, 1))
    ws = arena.carve("forward_workspace", (wsb,), dtype=torch.uint8)
    rc = []
    rep = run_checked(arena, "frozen_encoder_ex_forward(act_input=%d, tap=%d)" % (act, tap), lambda: rc.append(lib.snb200_frozen_encoder_ex_forward(
        b, n, act, x.data_ptr(), nconv, conv, npf, csz, pooled.data_ptr(), route.data_ptr(), tap, _vp(tap_out), _ptrs(zs), _addr(ws), wsb,
        None)), [ws], full=[pooled, route] + zs + ([tap_out] if tap_out is not None else []))
    for btap in sorted({tap, -1}, reverse=True):
        gp = arena.carve("grad_pooled.tap%d" % btap, (npf, b, C), fill=torch.randn(npf, b, C, generator=g))
        gtap = arena.carve("grad_tap.tap%d" % btap, tuple(tap_out.shape), fill=torch.randn(tuple(tap_out.shape), generator=g)) if btap >= 0 else None
        gin = arena.carve("grad_in.tap%d" % btap, (b, n, c_in))
        bwsb = int(lib.snb200_frozen_encoder_ex_backward_workspace_bytes(b, n, act, nconv, conv, npf, btap))
        bws = arena.carve("backward_workspace.tap%d" % btap, (bwsb,), dtype=torch.uint8)
        rep += run_checked(arena, "frozen_encoder_ex_backward(act_input=%d, tap=%d)" % (act, btap), lambda: rc.append(
            lib.snb200_frozen_encoder_ex_backward(b, n, act, x.data_ptr(), nconv, conv, npf, csz, pooled.data_ptr(), route.data_ptr(), _ptrs(zs), btap,
                                                  _vp(gtap), gp.data_ptr(), gin.data_ptr(), _addr(bws), bwsb, None)), [bws], full=[gin])
    assert all(r == 0 for r in rc), lib.snb200_last_error()
    assert_clean(rep)
