"""The stand-alone entry points snb200_encoder_forward + snb200_fc_head_forward run the generator's own pool and FC-head kernel, so
chained they must give bit for bit what snb200_generator_forward gives on its exact-fp32 path: outputs, pooled features, running
statistics and num_batches_tracked, in training and eval mode, over the row-group variants of the head, its K-chunked staging of a
1024-wide input, FC layers narrower than one 16-channel pass and an FC input width that is not a multiple of 4 (the head's weight
slices then need a padded row stride to keep their float4 reads aligned)."""
import copy

import pytest
import torch

M = 16   # sampled points: FC outputs of 3 * M


@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _net(sb, name):
    from samplenet_b200.samplenet import LayerTableGenerator
    if name == "samplenet":
        return sb.SampleNet(M, 128, group_size=8, input_shape="bnc", output_shape="bnc")
    if name == "reconstruction":
        return sb.ReconstructionSampleNet(M)
    if name == "classification":
        return sb.ClassificationSampleNet(M)
    if name == "mixed_fc":   # BatchNorm with and without ReLU; a 10-wide layer (less than one 16-channel pass, K not a multiple of 4)
        return LayerTableGenerator([3, 64, 128], [128, 48, 10, 3 * M], [1, 1, 0], [1, 0, 0], 1e-5, 0.1)
    assert name == "wide_feat"   # 1024 pooled channels: the head stages fc1's input in K chunks
    return LayerTableGenerator([3, 64, 128, 1024], [1024, 256, 3 * M], [1, 0], [1, 0], 1e-3, 0.5)


def _randomise(net, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                c = m.num_features
                m.weight.copy_(1 + 0.6 * torch.randn(c, generator=g))   # some negative scales: the pool then takes the minimum
                m.bias.copy_(0.2 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                m.running_var.copy_(0.5 + torch.rand(c, generator=g))
    return net


def _buffers(net):
    return {k: v for k, v in net.state_dict().items() if "running" in k or "num_batches" in k}


@pytest.mark.gpu
@pytest.mark.parametrize("b", [2, 5, 33, 70, 256])
@pytest.mark.parametrize("name", ["samplenet", "reconstruction", "classification", "mixed_fc", "wide_feat"])
def test_standalone_pair_equals_exact_fp32_generator(sb, name, b):
    n = 300
    base = _randomise(_net(sb, name), b).cuda()
    g = torch.Generator().manual_seed(1000 + b)
    cloud = torch.rand(b, n, 3, generator=g).cuda() - 0.5
    for training in (True, False):
        for layout in ("bnc", "bcn"):
            x = cloud if layout == "bnc" else cloud.permute(0, 2, 1).contiguous()
            for oti in (0, M):
                results = []
                for unfused in (True, False):
                    net = copy.deepcopy(base).train(training)
                    conv, fc = net._layer_specs()
                    with torch.no_grad():
                        if unfused:
                            out, feat = sb.ops.generator_forward_unfused(x, layout, conv, fc, training, oti)
                        else:
                            out, feat = sb.ops.generator_forward(x, layout, conv, fc, training, oti, exact_fp32=True)
                    torch.cuda.synchronize()
                    results.append((out, feat, _buffers(net)))
                case = (name, b, training, layout, oti)
                (o1, f1, s1), (o2, f2, s2) = results
                assert torch.isfinite(o1).all() and torch.isfinite(f1).all(), case
                assert torch.equal(f1, f2), case
                assert torch.equal(o1, o2), case
                assert s1.keys() == s2.keys()
                for k in s1:
                    assert torch.equal(s1[k], s2[k]), (case, k)
                    if "num_batches" in k:
                        assert int(s1[k]) == int(training), (case, k)
                    elif training:
                        assert not torch.equal(s1[k], _buffers(base)[k]), (case, k)   # the update ran


def test_fc_head_rejects_unaligned_input():
    """fc_head_forward reads an input whose width is a multiple of 4 as float4 rows: a pointer off the 16-byte grid is refused before
    any launch (the tables are fake, never dereferenced)."""
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib
    from samplenet_b200._lib import Layer
    lib = _lib.lib()
    fc = (Layer * 2)()
    for i, (cin, cout) in enumerate(((128, 64), (64, 3 * M))):
        fc[i].c_in, fc[i].c_out = cin, cout
        fc[i].weight, fc[i].bias = 0x100000 + 0x1000 * i, 0x200000 + 0x1000 * i
    b = 8
    need = lib.snb200_fc_head_workspace_bytes(b, 2, fc)
    rc = lib.snb200_fc_head_forward(b, 0x300004, 2, fc, 0, 0x400000, 0, 0x500000, need, None)
    msg = lib.snb200_last_error().decode()
    assert rc == -1 and msg.startswith("fc_head_forward:") and "aligned" in msg, (rc, msg)
