"""Host-side answers of the generator's C ABI, without a GPU: workspace sizes, the backward's envelope and the return code and
message prefix of every argument rejection.  The tables are fake (non-null, 16-byte aligned integers, never dereferenced) because every
call here returns before any launch or device allocation.  The expected values were recorded before the host code was
restructured and must not drift: callers size their buffers with these numbers."""
import ctypes

import pytest
import torch

BNC = 0
SKIP_HEAD, SKIP_CONV, EXACT_FP32, PER_LAYER, SEPARATE_HEAD = 2, 4, 1, 8, 16
M3 = 192   # 3 x 64 sampled points

_next_ptr = [0x10000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, bn, relu, eps=1e-5, momentum=0.1):
    """widths = [c_in, c_out of layer 0, c_out of layer 1, ...]; bn / relu: one flag per layer."""
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out = widths[i], widths[i + 1]
        L.weight, L.bias = _ptr(), _ptr()
        if bn[i]:
            L.bn_weight, L.bn_bias, L.bn_running_mean, L.bn_running_var, L.bn_num_batches_tracked = _ptr(), _ptr(), _ptr(), _ptr(), _ptr()
            L.bn_eps, L.bn_momentum = eps, momentum
        L.relu = int(relu[i])
    return arr


def _tables(name):
    if name == "registration":
        conv = _table([3, 64, 64, 64, 128, 128], [1] * 5, [1] * 5)
        fc = _table([128, 256, 256, 256, M3], [1, 1, 1, 0], [1, 1, 1, 0])
    elif name == "reconstruction":
        conv = _table([3, 64, 128, 128, 256, 128], [1] * 5, [1] * 5)
        fc = _table([128, 256, 256, 256, M3], [1, 1, 1, 0], [1, 1, 1, 0])
    else:   # TF-style: BatchNorm (decay 0.5, eps 1e-3) on every layer, the last FC layer included
        conv = _table([3, 64, 64, 64, 128, 128], [1] * 5, [1] * 5, 1e-3, 0.5)
        fc = _table([128, 256, 256, 256, M3], [1] * 4, [1] * 4, 1e-3, 0.5)
    return conv, fc


TABLES = ("registration", "reconstruction", "tf")
BATCHES = (1, 2, 7, 32, 37, 64, 128, 256)
POINTS = (77, 1000, 1024, 2048)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def _sm_count_is_default():
    """The backward's sizes and envelope depend on the SM count: 132 on an H100 SXM, and the fallback when no device is visible."""
    return not torch.cuda.is_available() or torch.cuda.get_device_properties(0).multi_processor_count == 132


# (table, B, N) -> (generator_workspace_bytes, generator_backward_workspace_bytes, encoder_workspace_bytes, generator_backward_supported)
EXPECTED_SIZES = {
    ('registration', 1, 77): (210176, 498944, 87040, 0),
    ('registration', 1, 1000): (1169664, 5407488, 1039360, 0),
    ('registration', 1, 1024): (1194240, 5435136, 1063936, 0),
    ('registration', 1, 2048): (2259200, 10858240, 2120704, 0),
    ('registration', 2, 77): (298240, 858112, 166912, 1),
    ('registration', 2, 1000): (2217216, 10675200, 2071552, 1),
    ('registration', 2, 1024): (2266368, 10863104, 2120704, 1),
    ('registration', 2, 2048): (4396288, 21709312, 4234240, 1),
    ('registration', 7, 77): (738560, 2917120, 566272, 1),
    ('registration', 7, 1000): (7454976, 36791040, 7232512, 1),
    ('registration', 7, 1024): (7627008, 37626112, 7404544, 1),
    ('registration', 7, 2048): (15081728, 50270464, 14801920, 1),
    ('registration', 32, 77): (2940160, 13212160, 2563072, 1),
    ('registration', 32, 1000): (33643776, 68480000, 33037312, 1),
    ('registration', 32, 1024): (34430208, 69266432, 33823744, 1),
    ('registration', 32, 2048): (68508928, 102820864, 67640320, 1),
    ('registration', 37, 77): (3380480, 15404800, 2962432, 1),
    ('registration', 37, 1000): (38881536, 73624320, 38198272, 1),
    ('registration', 37, 1024): (39790848, 74533632, 39107584, 1),
    ('registration', 37, 2048): (79194368, 113330944, 78208000, 1),
    ('registration', 64, 77): (5758208, 26327040, 5118976, 1),
    ('registration', 64, 1000): (67165440, 101403648, 66067456, 1),
    ('registration', 64, 1024): (68738304, 102976512, 67640320, 1),
    ('registration', 64, 2048): (136895744, 170085376, 135273472, 1),
    ('registration', 128, 77): (11394304, 46271488, 10230784, 0),
    ('registration', 128, 1000): (134208768, 167250944, 132127744, 0),
    ('registration', 128, 1024): (137354496, 170396672, 135273472, 0),
    ('registration', 128, 2048): (273669376, 304614400, 270539776, 0),
    ('registration', 256, 77): (22666496, 56986624, 20454400, 0),
    ('registration', 256, 1000): (268295424, 298945536, 264248320, 0),
    ('registration', 256, 1024): (274586880, 305236992, 270539776, 0),
    ('registration', 256, 2048): (547216640, 573672448, 541072384, 0),
    ('reconstruction', 1, 77): (358656, 1273088, 169984, 0),
    ('reconstruction', 1, 1000): (2263296, 13808384, 2067456, 0),
    ('reconstruction', 1, 1024): (2312448, 13860608, 2116608, 0),
    ('reconstruction', 1, 2048): (4425984, 27705088, 4221952, 0),
    ('reconstruction', 2, 77): (525568, 2171904, 328704, 0),
    ('reconstruction', 2, 1000): (4334848, 27242496, 4123648, 0),
    ('reconstruction', 2, 1024): (4433152, 27709952, 4221952, 0),
    ('reconstruction', 2, 2048): (8660224, 55398912, 8432640, 0),
    ('reconstruction', 7, 77): (1360128, 7389952, 1122304, 0),
    ('reconstruction', 7, 1000): (14692608, 94420736, 14404608, 0),
    ('reconstruction', 7, 1024): (15036672, 96579840, 14748672, 0),
    ('reconstruction', 7, 2048): (29831424, 125780224, 29486080, 0),
    ('reconstruction', 32, 77): (5532928, 33480192, 5090304, 0),
    ('reconstruction', 32, 1000): (66481408, 162077696, 65809408, 0),
    ('reconstruction', 32, 1024): (68054272, 163650560, 67382272, 0),
    ('reconstruction', 32, 2048): (135687424, 230759424, 134753280, 0),
    ('reconstruction', 37, 77): (6367488, 39062272, 5883904, 0),
    ('reconstruction', 37, 1000): (76839168, 172342016, 76090368, 0),
    ('reconstruction', 37, 1024): (78657792, 174160640, 77908992, 0),
    ('reconstruction', 37, 2048): (156858624, 251755264, 155806720, 0),
    ('reconstruction', 64, 77): (10874112, 66859008, 10169344, 0),
    ('reconstruction', 64, 1000): (132771072, 227769344, 131607552, 0),
    ('reconstruction', 64, 1024): (135916800, 230915072, 134753280, 0),
    ('reconstruction', 64, 2048): (271183104, 365132800, 269495296, 0),
    ('reconstruction', 128, 77): (21556480, 117193728, 20327424, 0),
    ('reconstruction', 128, 1000): (265350400, 359152640, 263203840, 0),
    ('reconstruction', 128, 1024): (271641856, 365444096, 269495296, 0),
    ('reconstruction', 128, 2048): (542174464, 633879552, 538979328, 0),
    ('reconstruction', 256, 77): (42921216, 138001408, 40643584, 0),
    ('reconstruction', 256, 1000): (530509056, 621919232, 526396416, 0),
    ('reconstruction', 256, 1024): (543091968, 634502144, 538979328, 0),
    ('reconstruction', 256, 2048): (1084157184, 1171373056, 1077947392, 0),
    ('tf', 1, 77): (210176, 498944, 87040, 0),
    ('tf', 1, 1000): (1169664, 5407488, 1039360, 0),
    ('tf', 1, 1024): (1194240, 5435136, 1063936, 0),
    ('tf', 1, 2048): (2259200, 10858240, 2120704, 0),
    ('tf', 2, 77): (298240, 858112, 166912, 1),
    ('tf', 2, 1000): (2217216, 10675200, 2071552, 1),
    ('tf', 2, 1024): (2266368, 10863104, 2120704, 1),
    ('tf', 2, 2048): (4396288, 21709312, 4234240, 1),
    ('tf', 7, 77): (738560, 2917120, 566272, 1),
    ('tf', 7, 1000): (7454976, 36791040, 7232512, 1),
    ('tf', 7, 1024): (7627008, 37626112, 7404544, 1),
    ('tf', 7, 2048): (15081728, 50270464, 14801920, 1),
    ('tf', 32, 77): (2940160, 13212160, 2563072, 1),
    ('tf', 32, 1000): (33643776, 68480000, 33037312, 1),
    ('tf', 32, 1024): (34430208, 69266432, 33823744, 1),
    ('tf', 32, 2048): (68508928, 102820864, 67640320, 1),
    ('tf', 37, 77): (3380480, 15404800, 2962432, 1),
    ('tf', 37, 1000): (38881536, 73624320, 38198272, 1),
    ('tf', 37, 1024): (39790848, 74533632, 39107584, 1),
    ('tf', 37, 2048): (79194368, 113330944, 78208000, 1),
    ('tf', 64, 77): (5758208, 26327040, 5118976, 1),
    ('tf', 64, 1000): (67165440, 101403648, 66067456, 1),
    ('tf', 64, 1024): (68738304, 102976512, 67640320, 1),
    ('tf', 64, 2048): (136895744, 170085376, 135273472, 1),
    ('tf', 128, 77): (11394304, 46271488, 10230784, 0),
    ('tf', 128, 1000): (134208768, 167250944, 132127744, 0),
    ('tf', 128, 1024): (137354496, 170396672, 135273472, 0),
    ('tf', 128, 2048): (273669376, 304614400, 270539776, 0),
    ('tf', 256, 77): (22666496, 56986624, 20454400, 0),
    ('tf', 256, 1000): (268295424, 298945536, 264248320, 0),
    ('tf', 256, 1024): (274586880, 305236992, 270539776, 0),
    ('tf', 256, 2048): (547216640, 573672448, 541072384, 0),
}
# (table, B) -> fc_head_workspace_bytes
EXPECTED_FC_HEAD = {
    ('registration', 1): 2048,
    ('registration', 2): 4096,
    ('registration', 7): 14336,
    ('registration', 32): 65536,
    ('registration', 37): 75776,
    ('registration', 64): 131072,
    ('registration', 128): 262144,
    ('registration', 256): 524288,
    ('reconstruction', 1): 2048,
    ('reconstruction', 2): 4096,
    ('reconstruction', 7): 14336,
    ('reconstruction', 32): 65536,
    ('reconstruction', 37): 75776,
    ('reconstruction', 64): 131072,
    ('reconstruction', 128): 262144,
    ('reconstruction', 256): 524288,
    ('tf', 1): 2048,
    ('tf', 2): 4096,
    ('tf', 7): 14336,
    ('tf', 32): 65536,
    ('tf', 37): 75776,
    ('tf', 64): 131072,
    ('tf', 128): 262144,
    ('tf', 256): 524288,
}


def _sizes(lib, name, b, n):
    conv, fc = _tables(name)
    return (lib.snb200_generator_workspace_bytes(b, n, 5, conv, 4, fc), lib.snb200_generator_backward_workspace_bytes(b, n, 5, conv, 4, fc),
            lib.snb200_encoder_workspace_bytes(b, n, 5, conv), lib.snb200_generator_backward_supported(b, n, 5, conv, 4, fc))


@pytest.mark.parametrize("name", TABLES)
def test_workspace_sizes_and_backward_envelope(lib, name):
    sm_default = _sm_count_is_default()
    for b in BATCHES:
        for n in POINTS:
            gen, bwd, enc, sup = _sizes(lib, name, b, n)
            want = EXPECTED_SIZES[(name, b, n)]
            assert (gen, enc) == (want[0], want[2]), (name, b, n)
            if sm_default:
                assert (bwd, sup) == (want[1], want[3]), (name, b, n)
        conv, fc = _tables(name)
        assert lib.snb200_fc_head_workspace_bytes(b, 4, fc) == EXPECTED_FC_HEAD[(name, b)], (name, b)


# ---------------------------------------------------------------------------------------------------- rejections
# Each case changes one argument of a call that would otherwise be valid.  Apart from the workspace case, the workspace is null: a check
# that went missing then ends in a workspace error instead of a launch on fake pointers.
def _nine(widths_from, kind):
    w = [widths_from] + [64] * 9
    return _table(w, [1] * 9, [1] * 9) if kind == "conv" else _table(w, [0] * 9, [0] * 9)


def _mutations():
    """kind -> function(args) that applies one bad argument to a dict of call arguments."""
    def set_(**kw):
        def f(a):
            a.update(kw)
        return f

    def layer(table, i, **kw):
        def f(a):
            for k, v in kw.items():
                setattr(a[table][i], k, v)
        return f

    return {
        "conv_null": set_(conv=None),
        "conv_empty": set_(nconv=0),
        "conv_nine": set_(conv=_nine(3, "conv"), nconv=9),
        "fc_null": set_(fc=None),
        "fc_empty": set_(nfc=0),
        "fc_nine": set_(fc=_nine(128, "fc"), nfc=9),
        "width_chain": layer("conv", 2, c_in=32),
        "bn_without_bias": layer("conv", 1, bn_bias=None),
        "fc_input_width": layer("fc", 0, c_in=64),
        "transpose_inner": set_(oti=5),
        "transpose_inner_negative": set_(oti=-3),
        "layout": set_(layout=7),
        "zsave_entry_null": lambda a: a["zsave"].__setitem__(3, None),
        "eval_no_running_conv": lambda a: (a.update(training=0), setattr(a["conv"][1], "bn_running_mean", None)),
        "eval_no_running_fc": lambda a: (a.update(training=0), setattr(a["fc"][0], "bn_running_var", None)),
        "train_bn_b1": set_(b=1),
        "b257": set_(b=257),
        "envelope_b65": set_(b=65),
        "envelope_no_relu": layer("conv", 2, relu=0),
        "flag_exact_fp32": set_(flags=EXACT_FP32),
        "flag_skip_head": set_(flags=SKIP_HEAD),
        "flag_skip_conv": set_(flags=SKIP_CONV),
        "flag_per_layer": set_(flags=PER_LAYER),
        "flag_separate_head": set_(flags=SEPARATE_HEAD),
    }


def _base(name):
    conv, fc = _tables(name)
    zs = (ctypes.c_void_p * 5)(*[_ptr() for _ in range(5)])
    return dict(b=32, n=1024, layout=BNC, conv=conv, nconv=5, fc=fc, nfc=4, training=1, oti=0, flags=0, zsave=zs, ws=None, wsb=0)


def _call(lib, entry, a):
    x, out, feat, g = _ptr(), _ptr(), _ptr(), _ptr()
    if entry == "generator_forward":
        return lib.snb200_generator_forward(a["b"], a["n"], BNC, x, a["nconv"], a["conv"], a["nfc"], a["fc"], a["training"], out, a["oti"], feat,
                                            a["flags"], a["ws"], a["wsb"], None)
    if entry == "generator_train_forward":
        return lib.snb200_generator_train_forward(a["b"], a["n"], a["layout"], x, a["nconv"], a["conv"], a["nfc"], a["fc"], out, a["oti"], feat, a["zsave"],
                                                  a["flags"], a["ws"], a["wsb"], None)
    if entry == "generator_backward":
        from samplenet_b200._lib import LayerGrad
        gconv, gfc = (LayerGrad * 9)(), (LayerGrad * 9)()
        return lib.snb200_generator_backward(a["b"], a["n"], a["layout"], x, a["nconv"], a["conv"], a["nfc"], a["fc"], a["zsave"], _ptr(), g, a["oti"],
                                             gconv, gfc, a["ws"], a["wsb"], None)
    if entry == "encoder_forward":
        return lib.snb200_encoder_forward(a["b"], a["n"], BNC, x, a["nconv"], a["conv"], a["training"], feat, a["ws"], a["wsb"], None)
    assert entry == "fc_head_forward"
    return lib.snb200_fc_head_forward(a["b"], x, a["nfc"], a["fc"], a["training"], out, a["oti"], a["ws"], a["wsb"], None)


def _need(lib, entry, a):
    if entry == "encoder_forward":
        return lib.snb200_encoder_workspace_bytes(a["b"], a["n"], a["nconv"], a["conv"])
    if entry == "fc_head_forward":
        return lib.snb200_fc_head_workspace_bytes(a["b"], a["nfc"], a["fc"])
    if entry == "generator_backward":
        return lib.snb200_generator_backward_workspace_bytes(a["b"], a["n"], a["nconv"], a["conv"], a["nfc"], a["fc"])
    return lib.snb200_generator_workspace_bytes(a["b"], a["n"], a["nconv"], a["conv"], a["nfc"], a["fc"])


_TABLE_KINDS = ["conv_null", "conv_empty", "conv_nine", "fc_null", "fc_empty", "fc_nine", "width_chain", "bn_without_bias"]
_ENVELOPE = ["envelope_b65", "envelope_no_relu"]
_FLAGS = ["flag_exact_fp32", "flag_skip_head", "flag_skip_conv", "flag_per_layer", "flag_separate_head"]
# entry point -> the bad arguments it rejects (conv-only / FC-only entry points see only their own table)
_TRAINING = ["transpose_inner", "transpose_inner_negative", "layout", "zsave_entry_null"]
REJECTIONS = {
    "generator_forward": _TABLE_KINDS + ["fc_input_width", "transpose_inner", "eval_no_running_conv", "eval_no_running_fc", "train_bn_b1", "b257",
                                         "workspace_short"],
    "generator_train_forward": _TABLE_KINDS + ["train_bn_b1", "b257", "workspace_short"] + _FLAGS + _ENVELOPE + _TRAINING,
    "generator_backward": _TABLE_KINDS + ["train_bn_b1", "b257", "workspace_short"] + _ENVELOPE + _TRAINING,
    "encoder_forward": [k for k in _TABLE_KINDS if not k.startswith("fc_")] + ["eval_no_running_conv", "workspace_short"],
    "fc_head_forward": [k for k in _TABLE_KINDS if k.startswith("fc_")] + ["transpose_inner", "eval_no_running_fc", "train_bn_b1", "b257",
                                                                           "workspace_short"],
}
# the FC-only entry point checks its own chain and BatchNorm pairs on the FC table
_FC_TABLE_FAULTS = {"width_chain": ("fc", 2, "c_in", 32), "bn_without_bias": ("fc", 1, "bn_bias", None)}
REJECTIONS["fc_head_forward"] += list(_FC_TABLE_FAULTS)

# (entry point, bad argument) -> return code: -1 SNB200_EINVAL, -2 SNB200_EWORKSPACE
EXPECTED_RC = {
    ('encoder_forward', 'conv_null'): -1,
    ('encoder_forward', 'conv_empty'): -1,
    ('encoder_forward', 'conv_nine'): -1,
    ('encoder_forward', 'width_chain'): -1,
    ('encoder_forward', 'bn_without_bias'): -1,
    ('encoder_forward', 'eval_no_running_conv'): -1,
    ('encoder_forward', 'workspace_short'): -2,
    ('fc_head_forward', 'fc_null'): -1,
    ('fc_head_forward', 'fc_empty'): -1,
    ('fc_head_forward', 'fc_nine'): -1,
    ('fc_head_forward', 'transpose_inner'): -1,
    ('fc_head_forward', 'eval_no_running_fc'): -1,
    ('fc_head_forward', 'train_bn_b1'): -1,
    ('fc_head_forward', 'b257'): -1,
    ('fc_head_forward', 'workspace_short'): -2,
    ('fc_head_forward', 'width_chain'): -1,
    ('fc_head_forward', 'bn_without_bias'): -1,
    ('generator_backward', 'conv_null'): -1,
    ('generator_backward', 'conv_empty'): -1,
    ('generator_backward', 'conv_nine'): -1,
    ('generator_backward', 'fc_null'): -1,
    ('generator_backward', 'fc_empty'): -1,
    ('generator_backward', 'fc_nine'): -1,
    ('generator_backward', 'width_chain'): -1,
    ('generator_backward', 'bn_without_bias'): -1,
    ('generator_backward', 'train_bn_b1'): -1,
    ('generator_backward', 'b257'): -1,
    ('generator_backward', 'workspace_short'): -2,
    ('generator_backward', 'envelope_b65'): -1,
    ('generator_backward', 'envelope_no_relu'): -1,
    ('generator_forward', 'conv_null'): -1,
    ('generator_forward', 'conv_empty'): -1,
    ('generator_forward', 'conv_nine'): -1,
    ('generator_forward', 'fc_null'): -1,
    ('generator_forward', 'fc_empty'): -1,
    ('generator_forward', 'fc_nine'): -1,
    ('generator_forward', 'width_chain'): -1,
    ('generator_forward', 'bn_without_bias'): -1,
    ('generator_forward', 'fc_input_width'): -1,
    ('generator_forward', 'transpose_inner'): -1,
    ('generator_forward', 'eval_no_running_conv'): -1,
    ('generator_forward', 'eval_no_running_fc'): -1,
    ('generator_forward', 'train_bn_b1'): -1,
    ('generator_forward', 'b257'): -1,
    ('generator_forward', 'workspace_short'): -2,
    ('generator_train_forward', 'conv_null'): -1,
    ('generator_train_forward', 'conv_empty'): -1,
    ('generator_train_forward', 'conv_nine'): -1,
    ('generator_train_forward', 'fc_null'): -1,
    ('generator_train_forward', 'fc_empty'): -1,
    ('generator_train_forward', 'fc_nine'): -1,
    ('generator_train_forward', 'width_chain'): -1,
    ('generator_train_forward', 'bn_without_bias'): -1,
    ('generator_train_forward', 'train_bn_b1'): -1,
    ('generator_train_forward', 'b257'): -1,
    ('generator_train_forward', 'workspace_short'): -2,
    ('generator_train_forward', 'flag_exact_fp32'): -1,
    ('generator_train_forward', 'flag_skip_head'): -1,
    ('generator_train_forward', 'flag_skip_conv'): -1,
    ('generator_train_forward', 'flag_per_layer'): -1,
    ('generator_train_forward', 'flag_separate_head'): -1,
    ('generator_train_forward', 'envelope_b65'): -1,
    ('generator_train_forward', 'envelope_no_relu'): -1,
    # the training entries of both routes share one set of checks
    ('generator_train_forward', 'transpose_inner'): -1,
    ('generator_train_forward', 'transpose_inner_negative'): -1,
    ('generator_train_forward', 'layout'): -1,
    ('generator_train_forward', 'zsave_entry_null'): -1,
    ('generator_backward', 'transpose_inner'): -1,
    ('generator_backward', 'transpose_inner_negative'): -1,
    ('generator_backward', 'layout'): -1,
    ('generator_backward', 'zsave_entry_null'): -1,
}


def _rejection_rc(lib, entry, kind):
    a = _base("registration")
    if kind == "workspace_short":
        need = _need(lib, entry, a)
        a.update(ws=_ptr(), wsb=need - 1)
    elif entry == "fc_head_forward" and kind in _FC_TABLE_FAULTS:
        t, i, field, v = _FC_TABLE_FAULTS[kind]
        setattr(a[t][i], field, v)
    else:
        _mutations()[kind](a)
    rc = _call(lib, entry, a)
    msg = lib.snb200_last_error().decode()
    return rc, msg


@pytest.mark.parametrize("entry", sorted(REJECTIONS))
def test_rejections(lib, entry):
    for kind in REJECTIONS[entry]:
        rc, msg = _rejection_rc(lib, entry, kind)
        assert rc == EXPECTED_RC[(entry, kind)], (entry, kind, rc, msg)
        assert msg.startswith(entry + ":"), (entry, kind, msg)
