"""Schema-driven proto codec: text + binary wire format, reference prototxt goldens, V0 upgrade."""
import glob
import os

import numpy as np
import pytest

from poseidon_b200 import proto as P
from poseidon_b200.proto import parse_text, to_text

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")   # the reference's prototxt files


def test_text_roundtrip_and_defaults():
    txt = '''
    name: "n"  # comment
    layers { name: "c1" type: CONVOLUTION bottom: "data" top: "c1" blobs_lr: 1 blobs_lr: 2
      convolution_param { num_output: 8 kernel_size: 3 weight_filler { type: "gaussian" std: 0.01 } } }
    layers { name: 'r' type: RELU bottom: "c1" top: "c1" relu_param { negative_slope: 1e-1 } }
    input: "data" input_dim: 1 input_dim: 3 input_dim: 8 input_dim: 8
    '''
    net = parse_text(txt, P.NetParameter)
    assert net.name == "n" and len(net.layers) == 2
    l = net.layers[0]
    assert l.type == P.LayerType["CONVOLUTION"] and l.enum_name("type") == "CONVOLUTION"
    assert list(l.blobs_lr) == [1.0, 2.0]
    cp = l.convolution_param
    assert cp.num_output == 8 and cp.stride == 1 and cp.group == 1 and cp.bias_term is True      # defaults
    assert abs(cp.weight_filler.std - 0.01) < 1e-9 and cp.weight_filler.type == "gaussian"
    assert not cp.has("pad") and cp.pad == 0
    assert abs(net.layers[1].relu_param.negative_slope - 0.1) < 1e-7
    again = parse_text(to_text(net), P.NetParameter)
    assert again == net


def test_binary_roundtrip_packed_floats_and_unknown_fields():
    b = P.BlobProto(num=2, channels=3, height=1, width=2)
    b.data = np.arange(12, dtype=np.float32)
    b.diff = -np.arange(12, dtype=np.float32)
    raw = b.SerializeToString()
    # field 5, wire type 2 (packed), 48 bytes
    assert bytes([5 << 3 | 2, 48]) in raw
    b2 = P.BlobProto.FromString(raw)
    assert np.array_equal(b2.data, b.data) and np.array_equal(b2.diff, b.diff) and b2.channels == 3
    assert b2.blob_mode == 1 and b2.global_id == -1                              # defaults
    # unknown field (number 99, varint) is skipped
    raw2 = raw + bytes([0x98, 0x06, 0x2A])
    assert np.array_equal(P.BlobProto.FromString(raw2).data, b.data)
    # unpacked encoding of a packed field must also parse
    import struct
    unpacked = b"".join(bytes([5 << 3 | 5]) + struct.pack("<f", v) for v in (1.5, 2.5))
    assert list(P.BlobProto.FromString(unpacked).data) == [1.5, 2.5]


def test_nested_netparameter_binary_roundtrip():
    net = P.NetParameter(name="m")
    l = net.layers.add(name="ip", type="INNER_PRODUCT")
    l.bottom, l.top = ["x"], ["y"]
    l.blobs.append(P.array_to_blob(np.random.randn(4, 5).astype(np.float32)))
    l.blobs.append(P.array_to_blob(np.random.randn(4).astype(np.float32)))
    l.mutable("inner_product_param").num_output = 4
    st = P.SolverState(iter=7, learned_net="a.caffemodel")
    st.history.append(l.blobs[0].copy())
    for msg, cls in ((net, P.NetParameter), (st, P.SolverState)):
        again = cls.FromString(msg.SerializeToString())
        assert again == msg
    b = P.NetParameter.FromString(net.SerializeToString()).layers[0].blobs[0]
    assert (b.num, b.channels, b.height, b.width) == (1, 1, 4, 5)                   # Caffe IP weight shape
    sv = P.SVProto(layer_id=3)
    sv.a, sv.b = [1.0, 2.0], [3.0]
    sv2 = P.SVProto.FromString(sv.SerializeToString())
    assert list(sv2.a) == [1.0, 2.0] and list(sv2.b) == [3.0] and sv2.layer_id == 3


def test_negative_int_and_int64():
    sp = P.SolverParameter(random_seed=-1, max_iter=5)
    sp2 = P.SolverParameter.FromString(sp.SerializeToString())
    assert sp2.random_seed == -1 and sp2.max_iter == 5
    b = P.BlobProto(global_id=-7)
    assert P.BlobProto.FromString(b.SerializeToString()).global_id == -7


def test_parse_every_reference_prototxt():
    files = glob.glob(REF + "/models/*/*.prototxt") + glob.glob(REF + "/examples/*/*.prototxt")
    assert len(files) >= 20
    for f in files:
        with open(f) as fh:
            txt = fh.read()
        cls = P.SolverParameter if "solver" in os.path.basename(f) else P.NetParameter
        msg = parse_text(txt, cls)
        assert parse_text(to_text(msg), cls) == msg, f
    g = P.read_net(REF + "/models/bvlc_googlenet/train_test.prototxt")
    types = [l.enum_name("type") for l in g.layers]
    assert types.count("CONVOLUTION") == 59 and types.count("INNER_PRODUCT") == 5 and types.count("CONCAT") == 9


def test_v0_upgrade_with_padding_fold():
    txt = '''
    name: "v0" input: "data" input_dim: 1 input_dim: 3 input_dim: 9 input_dim: 9
    layers { layer { name: "pad1" type: "padding" pad: 2 } bottom: "data" top: "pad1" }
    layers { layer { name: "conv1" type: "conv" num_output: 4 kernelsize: 5 stride: 1
             weight_filler { type: "gaussian" std: 0.01 } blobs_lr: 1 blobs_lr: 2 } bottom: "pad1" top: "conv1" }
    layers { layer { name: "relu1" type: "relu" } bottom: "conv1" top: "conv1" }
    layers { layer { name: "pool1" type: "pool" pool: MAX kernelsize: 3 stride: 2 } bottom: "conv1" top: "pool1" }
    layers { layer { name: "fc" type: "innerproduct" num_output: 10 } bottom: "pool1" top: "fc" }
    '''
    from poseidon_b200.net.upgrade import upgrade_net_as_needed
    net = upgrade_net_as_needed(parse_text(txt, P.NetParameter))
    assert [l.enum_name("type") for l in net.layers] == ["CONVOLUTION", "RELU", "POOLING", "INNER_PRODUCT"]
    c = net.layers[0]
    assert c.convolution_param.pad == 2 and list(c.bottom) == ["data"] and c.convolution_param.kernel_size == 5
    assert list(c.blobs_lr) == [1.0, 2.0]
    assert net.layers[2].pooling_param.enum_name("pool") == "MAX" and net.layers[2].pooling_param.stride == 2


def test_legacy_data_transform_upgrade():
    txt = 'layers { name: "d" type: DATA top: "data" top: "label" data_param { source: "x" batch_size: 4 scale: 0.5 crop_size: 7 mirror: true } }'
    from poseidon_b200.net.upgrade import upgrade_net_as_needed
    net = upgrade_net_as_needed(parse_text(txt, P.NetParameter))
    tp = net.layers[0].transform_param
    assert tp.scale == 0.5 and tp.crop_size == 7 and tp.mirror is True
    assert not net.layers[0].data_param.has("scale")


def test_malformed_wire_data_raises_decode_error():
    """Mutated .caffemodel-style bytes: a clean parse or DecodeError (a ValueError) — nothing else, and no hang."""
    import numpy as np
    from poseidon_b200.models import zoo
    from test_host_fuzz import _mutations
    raw = zoo.lenet(batch=4, test_batch=4).SerializeToString()
    assert P.NetParameter.FromString(raw).SerializeToString() == raw
    rng = np.random.RandomState(0)
    seen = {"ok": 0, "err": 0}
    for mut in _mutations(raw, rng, 600):
        try:
            P.NetParameter.FromString(mut)
            seen["ok"] += 1
        except P.DecodeError:
            seen["err"] += 1
    assert seen["err"] > 100 and seen["ok"] > 50, seen


def test_malformed_prototxt_raises_parse_error():
    import numpy as np
    from poseidon_b200.models import zoo
    from test_host_fuzz import _mutations
    txt = P.to_text(zoo.lenet(batch=4, test_batch=4)).encode()
    rng = np.random.RandomState(0)
    seen = {"ok": 0, "err": 0}
    for mut in _mutations(txt, rng, 500):
        try:
            P.parse_text(mut.decode("utf-8", "replace"), P.NetParameter)
            seen["ok"] += 1
        except P.ParseError as e:
            assert "NetParameter" in str(e)
            seen["err"] += 1
    assert seen["err"] > 300, seen
    with pytest.raises(P.ParseError, match="bogus_field|unknown|no field"):
        P.parse_text('name: "x" bogus_field: 3', P.NetParameter)
