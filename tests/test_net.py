"""Net construction from Caffe definitions: zoo shapes, filtering, in-place, sharing, loss weights, IO."""
import pytest
import torch

from poseidon_b200 import Net
from poseidon_b200 import proto as P
from poseidon_b200.models import zoo
from poseidon_b200.proto import parse_text


def test_alexnet_shapes_and_params():
    net = Net(zoo.alexnet(batch=2, test_batch=2), phase=P.TRAIN)
    bs = net.blob_shapes
    assert bs["data"] == (2, 3, 227, 227) and bs["conv1"] == (2, 96, 55, 55) and bs["pool1"] == (2, 96, 27, 27)
    assert bs["conv2"] == (2, 256, 27, 27) and bs["pool2"] == (2, 256, 13, 13) and bs["pool5"] == (2, 256, 6, 6)
    assert tuple(net.layer_by_name["fc6"].weight.shape) == (4096, 9216)
    assert tuple(net.layer_by_name["conv2"].weight.shape) == (256, 48, 5, 5)
    assert net.num_params() == 60965224
    assert "accuracy" not in net.layer_names                      # TEST-only layer filtered out
    assert net.output_names == ["loss"]
    tn = Net(zoo.alexnet(batch=2, test_batch=2), phase=P.TEST)
    assert set(tn.output_names) == {"accuracy", "loss"}


def test_googlenet_structure():
    net = Net(zoo.googlenet(batch=1, test_batch=1), phase=P.TRAIN)
    types = [l.type_name for l in net.layers]
    assert types.count("CONVOLUTION") == 59 and types.count("INNER_PRODUCT") == 5 and types.count("CONCAT") == 9
    assert net.blob_shapes["inception_3a/output"] == (1, 256, 28, 28)
    assert net.blob_shapes["inception_5b/output"] == (1, 1024, 7, 7)
    assert net.blob_shapes["pool5/7x7_s1"] == (1, 1024, 1, 1)
    assert net.output_names == ["loss1/loss1", "loss2/loss1", "loss3/loss3"]
    w = {t: lw for tn, lws in zip(net.top_names, net.loss_weights) for t, lw in zip(tn, lws)}
    assert w["loss1/loss1"] == pytest.approx(0.3) and w["loss3/loss3"] == 1.0


def test_caffenet_vs_alexnet_ordering_and_vgg():
    c = Net(zoo.caffenet(batch=1, test_batch=1), phase=P.TRAIN)
    assert c.layer_names.index("pool1") < c.layer_names.index("norm1")
    a = Net(zoo.alexnet(batch=1, test_batch=1), phase=P.TRAIN)
    assert a.layer_names.index("norm1") < a.layer_names.index("pool1")
    v = zoo.vgg16(batch=1)
    assert sum(1 for l in v.layers if l.enum_name("type") == "CONVOLUTION") == 13


def test_forward_backward_small_net_cpu():
    txt = '''
    input: "data" input_dim: 4 input_dim: 3 input_dim: 12 input_dim: 12
    input: "label" input_dim: 4 input_dim: 1 input_dim: 1 input_dim: 1
    layers { name: "c" type: CONVOLUTION bottom: "data" top: "c" convolution_param { num_output: 6 kernel_size: 3 group: 1
             weight_filler { type: "xavier" } } }
    layers { name: "r" type: RELU bottom: "c" top: "c" }
    layers { name: "p" type: POOLING bottom: "c" top: "p" pooling_param { pool: MAX kernel_size: 3 stride: 2 } }
    layers { name: "n" type: LRN bottom: "p" top: "n" lrn_param { local_size: 3 alpha: 0.1 } }
    layers { name: "s" type: SPLIT bottom: "n" top: "n1" top: "n2" }
    layers { name: "f1" type: INNER_PRODUCT bottom: "n1" top: "f1" inner_product_param { num_output: 5 weight_filler { type: "gaussian" std: 0.1 } } }
    layers { name: "f2" type: INNER_PRODUCT bottom: "n2" top: "f2" inner_product_param { num_output: 5 weight_filler { type: "gaussian" std: 0.1 } } }
    layers { name: "e" type: ELTWISE bottom: "f1" bottom: "f2" top: "e" eltwise_param { operation: SUM coeff: 1 coeff: -0.5 } }
    layers { name: "loss" type: SOFTMAX_LOSS bottom: "e" bottom: "label" top: "loss" loss_weight: 2 }
    '''
    net = Net(parse_text(txt, P.NetParameter), phase=P.TRAIN)
    assert net.blob_shapes["p"] == (4, 6, 5, 5)          # ceil((10-3)/2)+1
    x = torch.randn(4, 3, 12, 12)
    y = torch.randint(0, 5, (4, 1, 1, 1)).float()
    loss, outs = net.forward({"data": x, "label": y})
    assert loss.item() == pytest.approx(2 * outs["loss"].item(), rel=1e-6)
    loss.backward()
    assert all(p.grad is not None for p in net.params)


def test_param_sharing_and_frozen_params():
    txt = '''
    input: "a" input_dim: 2 input_dim: 4 input_dim: 1 input_dim: 1
    input: "b" input_dim: 2 input_dim: 4 input_dim: 1 input_dim: 1
    layers { name: "ip1" type: INNER_PRODUCT bottom: "a" top: "o1" param: "w" param: "bias" blobs_lr: 1 blobs_lr: 0
             inner_product_param { num_output: 3 weight_filler { type: "gaussian" std: 1 } } }
    layers { name: "ip2" type: INNER_PRODUCT bottom: "b" top: "o2" param: "w" param: "bias"
             inner_product_param { num_output: 3 } }
    layers { name: "l" type: EUCLIDEAN_LOSS bottom: "o1" bottom: "o2" top: "l" }
    '''
    net = Net(parse_text(txt, P.NetParameter), phase=P.TRAIN)
    assert len(net.params) == 2
    assert net.layer_by_name["ip1"].weight is net.layer_by_name["ip2"].weight
    assert net.params[1].requires_grad is False and net.params_lr == [1.0, 0.0]
    a = torch.randn(2, 4, 1, 1)
    loss, _ = net.forward({"a": a, "b": a})
    assert loss.item() == pytest.approx(0.0, abs=1e-9)


def test_include_exclude_rules_levels_and_stages():
    txt = '''
    input: "x" input_dim: 1 input_dim: 2 input_dim: 1 input_dim: 1
    layers { name: "a" type: RELU bottom: "x" top: "a" include { phase: TRAIN } }
    layers { name: "b" type: RELU bottom: "x" top: "b" include { stage: "deploy" } }
    layers { name: "c" type: RELU bottom: "x" top: "c" exclude { min_level: 2 } }
    layers { name: "d" type: RELU bottom: "x" top: "d" include { phase: TEST not_stage: "deploy" } }
    '''
    p = parse_text(txt, P.NetParameter)
    assert Net(p, phase=P.TRAIN).layer_names == ["a", "c"]
    assert Net(p, phase=P.TEST).layer_names == ["c", "d"]
    assert Net(p, phase=P.TEST, stages=["deploy"]).layer_names == ["b", "c"]
    assert Net(p, phase=P.TRAIN, level=2).layer_names == ["a"]


def test_caffemodel_roundtrip_by_layer_name(tmp_path):
    net = Net(zoo.lenet(batch=2, test_batch=2), phase=P.TRAIN)
    path = str(tmp_path / "m.caffemodel")
    P.write_binary(path, net.to_proto())
    msg = P.read_binary(path, P.NetParameter)
    ip1 = [l for l in msg.layers if l.name == "ip1"][0]
    assert (ip1.blobs[0].num, ip1.blobs[0].channels, ip1.blobs[0].height, ip1.blobs[0].width) == (1, 1, 500, 800)
    assert (ip1.blobs[1].height, ip1.blobs[1].width) == (1, 500)
    conv1 = [l for l in msg.layers if l.name == "conv1"][0]
    assert (conv1.blobs[0].num, conv1.blobs[0].channels, conv1.blobs[0].height) == (20, 1, 5)
    net2 = Net(zoo.lenet(batch=2, test_batch=2), phase=P.TEST)
    loaded = net2.copy_trained_layers_from(path)
    assert set(loaded) == {"conv1", "conv2", "ip1", "ip2"}
    for a, b in zip(net.params, net2.params):
        assert torch.equal(a, b)


def test_errors():
    with pytest.raises(ValueError, match="Unknown blob input"):
        Net(parse_text('layers { name: "r" type: RELU bottom: "nope" top: "r" }', P.NetParameter))
    with pytest.raises(ValueError, match="takes 1 bottom"):
        Net(parse_text('input: "x" input_dim: 1 input_dim: 1 input_dim: 1 input_dim: 1 '
                       'layers { name: "r" type: RELU bottom: "x" bottom: "x" top: "r" }', P.NetParameter))


REF = __import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "golden", "reference")


@pytest.mark.parametrize("model,ref_net,ref_solver", [
    ("alexnet", "models/bvlc_alexnet/train_val.prototxt", "models/bvlc_alexnet/solver.prototxt"),
    ("caffenet", "models/bvlc_reference_caffenet/train_val.prototxt", "models/bvlc_reference_caffenet/solver.prototxt"),
    ("googlenet", "models/bvlc_googlenet/train_test.prototxt", "models/bvlc_googlenet/quick_solver.prototxt"),
])
def test_zoo_matches_reference_prototxt(model, ref_net, ref_solver):
    """Golden parity: the zoo builders produce the same graph as the reference's shipped model files — layer for layer
    (name, type, tops, blob shapes, parameter shapes, lr / decay multipliers, loss weights) — and the same solver."""
    import os
    ref_np = P.read_net(os.path.join(REF, ref_net))
    for phase in (P.TRAIN, P.TEST):
        ours = Net(zoo.get_model(model), phase=phase)
        theirs = Net(ref_np, phase=phase)
        assert ours.layer_names == theirs.layer_names
        assert [l.type_name for l in ours.layers] == [l.type_name for l in theirs.layers]
        assert ours.top_names == theirs.top_names and ours.bottom_names == theirs.bottom_names
        assert {k: v[1:] for k, v in ours.blob_shapes.items()} == {k: v[1:] for k, v in theirs.blob_shapes.items()}
        for a, b in zip(ours.layers, theirs.layers):
            assert [tuple(p.shape) for p in a.blobs] == [tuple(p.shape) for p in b.blobs], a.layer_name
        assert ours.loss_weights == theirs.loss_weights
        assert ours.params_lr == theirs.params_lr and ours.params_weight_decay == theirs.params_weight_decay
    a, b = zoo.MODELS[model][1](), P.read_solver(os.path.join(REF, ref_solver))
    # (`display` is left out: the reference's CaffeNet solver ships a debugging leftover, "display: 1 #20")
    for f in ("base_lr", "lr_policy", "gamma", "stepsize", "power", "momentum", "weight_decay", "max_iter",
              "test_interval", "snapshot"):
        assert getattr(a, f) == pytest.approx(getattr(b, f)) if isinstance(getattr(b, f), float) else getattr(a, f) == getattr(b, f), f
    assert list(a.test_iter) == list(b.test_iter)


def test_deploy_nets_match_reference_and_share_weights_by_name(tmp_path):
    """zoo.deploy(): the generated AlexNet / CaffeNet deploy nets have the reference deploy.prototxt's layers (names,
    types, bottoms / tops, parameters); a deploy net loads a .caffemodel of its train_val net by name and reproduces
    the TEST-phase class probabilities."""
    import os
    import torch
    from poseidon_b200.models import zoo
    for ours, ref in (("alexnet", "bvlc_alexnet"), ("caffenet", "bvlc_reference_caffenet")):
        path = os.path.join(REF, "models", ref, "deploy.prototxt")
        want = P.read_net(path)
        got = zoo.deploy(zoo.MODELS[ours][0]())
        assert list(got.input) == list(want.input) and list(got.input_dim) == list(want.input_dim)
        assert [(l.name, l.enum_name("type"), list(l.bottom), list(l.top)) for l in got.layers] == \
               [(l.name, l.enum_name("type"), list(l.bottom), list(l.top)) for l in want.layers]
        for a, b in zip(got.layers, want.layers):
            for f in ("convolution_param", "pooling_param", "lrn_param", "inner_product_param", "dropout_param"):
                if b.has(f):
                    ga, gb = getattr(a, f), getattr(b, f)
                    for k in ("num_output", "kernel_size", "stride", "pad", "group", "pool", "local_size", "alpha", "beta",
                              "dropout_ratio"):
                        if hasattr(gb, k) and gb.has(k):
                            va, vb = getattr(ga, k), getattr(gb, k)
                            same = abs(va - vb) <= 1e-6 * abs(vb) if isinstance(vb, float) else va == vb
                            assert same, (a.name, f, k, va, vb)
    # weights by name + identical probabilities (LeNet, small)
    train = zoo.lenet(batch=4, test_batch=4)
    tnet = Net(train, phase=P.TEST)
    P.write_binary(str(tmp_path / "w.caffemodel"), tnet.to_proto())
    dnet = Net(zoo.deploy(train, batch=4), phase=P.TEST)
    dnet.copy_trained_layers_from(str(tmp_path / "w.caffemodel"))
    x = torch.rand(4, 1, 28, 28)
    _, out = dnet.forward({"data": x})
    # run the train_val net's layers by hand on the same input: conv1..ip2 then softmax
    blobs = {"data": x * 1.0}
    for name, layer, bn, tn in zip(tnet.layer_names, tnet.layers, tnet.bottom_names, tnet.top_names):
        if layer.type_name in ("DATA", "ACCURACY", "SOFTMAX_LOSS"):
            continue
        outs = layer(*[blobs[b] for b in bn])
        for t, o in zip(tn, outs):
            blobs[t] = o
    want_prob = torch.softmax(blobs["ip2"].reshape(4, -1), 1)
    assert torch.allclose(out["prob"].reshape(4, -1), want_prob, atol=1e-6)
    assert "accuracy" not in dnet.layer_names and "loss" not in dnet.layer_names
    # GoogLeNet: auxiliary classifiers are pruned, the main path ends in prob
    g = zoo.deploy(zoo.googlenet(batch=2, test_batch=2))
    names = [l.name for l in g.layers]
    assert not any(n.startswith("loss1/") or n.startswith("loss2/") for n in names) and names[-1] == "prob"
    assert g.layers[-1].bottom[0] == "loss3/classifier"
