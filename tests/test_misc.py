"""Smaller API-parity pieces: split insertion, flag context, sufficient-vector containers, SFB cost model."""
import torch

from poseidon_b200 import Net
from poseidon_b200 import proto as P
from poseidon_b200.proto import parse_text


def test_insert_splits_names_and_equivalence():
    from poseidon_b200.net.insert_splits import insert_splits
    txt = '''input: "x" input_dim: 2 input_dim: 3 input_dim: 1 input_dim: 1
    layers { name: "a" type: POWER bottom: "x" top: "a" power_param { scale: 2 } }
    layers { name: "b" type: RELU bottom: "a" top: "b" }
    layers { name: "c" type: SIGMOID bottom: "a" top: "c" }
    layers { name: "e" type: ELTWISE bottom: "b" bottom: "c" top: "e" }'''
    p = parse_text(txt, P.NetParameter)
    o = insert_splits(p)
    names = [l.name for l in o.layers]
    assert names == ["a", "a_a_0_split", "b", "c", "e"]
    assert list(o.layers[1].top) == ["a_a_0_split_0", "a_a_0_split_1"]
    x = torch.randn(2, 3, 1, 1)
    _, o1 = Net(p).forward({"x": x})
    _, o2 = Net(o).forward({"x": x})
    assert torch.allclose(o1["e"], o2["e"])


def test_context_flag_store():
    from poseidon_b200.utils.context import Context
    c = Context().load({"num_table_threads": 5, "svb": "true", "table_staleness": 2, "lr": "0.5", "none": None})
    assert c.get_int32("table_staleness") == 2 and c.get_bool("svb") and c.get_double("lr") == 0.5
    assert c.get_int32("num_app_threads") == 4
    assert Context.parse_int_list("0,1, 3") == [0, 1, 3]
    assert Context.get_instance() is Context.get_instance()


def test_sufficient_vector_roundtrip_and_queue():
    from poseidon_b200.parallel.sfb import SufficientVector, SufficientVectorQueue, sfb_bytes, sfb_wins
    a, b = torch.randn(4, 3), torch.randn(4, 5)
    sv = SufficientVector(a, b, layer_id=7)
    raw = sv.to_proto().SerializeToString()
    sv2 = SufficientVector.from_proto(P.SVProto.FromString(raw), (4, 3), (4, 5))
    assert sv2.layer_id == 7 and torch.allclose(sv2.gradient(), a.t() @ b, atol=1e-6)
    q = SufficientVectorQueue(max_read_count=2)
    q.add(sv)
    assert q.get() is sv and len(q) == 1      # first reader: still queued
    assert q.get() is sv and len(q) == 0      # second reader retires it
    assert q.get() is None
    # cost model (SURVEY 7.3 #2): AlexNet b=256, P=8
    assert sfb_wins(256, 4096, 9216, 8) and sfb_wins(256, 4096, 4096, 8) and not sfb_wins(256, 1000, 4096, 8)
    assert sfb_wins(64, 4096, 25088, 8)                             # VGG-16 fc6
    by = sfb_bytes(256, 4096, 9216, 8, 4)
    assert by["sfb_egress"] == 256 * (4096 + 9216) * 4


def test_stats_and_timer(tmp_path):
    from poseidon_b200.utils.stats import Stats
    from poseidon_b200.utils.timer import Timer
    st = Stats()
    with st.timer("x"):
        pass
    st.count("n", 3)
    st.set("bytes", {"a": 1})
    st.dump_yaml(str(tmp_path / "s.yaml"))
    import yaml
    d = yaml.safe_load((tmp_path / "s.yaml").read_text())
    assert d["counters"]["n"] == 3 and d["timer_calls"]["x"] == 1
    t = Timer("cpu")
    t.start()
    t.stop()
    assert t.milliseconds() >= 0


def test_hostfile_parser(tmp_path):
    from poseidon_b200.parallel.context import parse_hostfile
    f = tmp_path / "hosts"
    f.write_text("# comment\n1 10.0.0.2 9999\n0 127.0.0.1 9999\n")
    assert parse_hostfile(str(f)) == [(0, "127.0.0.1", 9999), (1, "10.0.0.2", 9999)]


def test_fault_injection_directives(monkeypatch):
    import time
    from poseidon_b200.utils import fault
    assert fault.parse("delay:rank=1,step=3,ms=20; kill:rank=2,step=5") == [
        ("delay", {"rank": 1, "step": 3, "ms": 20}), ("kill", {"rank": 2, "step": 5})]
    monkeypatch.setenv("POSEIDON_FAULT", "delay:rank=0,step=2,ms=30;raise:rank=0,step=4")
    fault.reset()
    t0 = time.time(); fault.maybe_inject(0, 1); assert time.time() - t0 < 0.02
    t0 = time.time(); fault.maybe_inject(0, 2); assert time.time() - t0 >= 0.03
    fault.maybe_inject(1, 4)                       # other rank: nothing
    try:
        fault.maybe_inject(0, 4)
        raise AssertionError("expected the injected fault")
    except RuntimeError as e:
        assert "injected fault" in str(e)
    monkeypatch.delenv("POSEIDON_FAULT")
    fault.reset()


def test_nvtx_ranges_are_noops_without_cuda():
    from poseidon_b200.utils import trace
    with trace.nvtx_range("x"):
        pass


def test_bench_harness_self_test_on_cpu():
    """bench.py --allow-cpu: the whole harness (device-resident leg, end-to-end leg with deferred loss reads, JSON contract)
    runs on a GPU-less box; numbers are meaningless, the control flow and the output keys are what is checked."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--allow-cpu", "--model", "lenet", "--steps", "3",
                          "--warmup", "3"], capture_output=True, text=True, timeout=300, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "clocks", "gpu_launches", "e2e"):
        assert k in d, k
    assert d["steps"] == 3 and d["warmup"] == 3 and d["n_gpus"] == 1 and d["value"] > 0
    assert d["e2e"]["value"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] == 4
    ref = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference"], capture_output=True,
                         text=True, timeout=120, cwd=root)
    r = json.loads(ref.stdout.strip().splitlines()[-1])
    assert r["impl"] == "reference" and "unavailable" in r


def test_caffe_root_placeholder_and_relative_paths(tmp_path, monkeypatch):
    """The reference's shipped prototxts spell paths as CAFFE_ROOT/...; they load without hand-editing."""
    from poseidon_b200.utils import paths
    monkeypatch.setattr(paths, "_root_hint", None)
    monkeypatch.delenv("CAFFE_ROOT", raising=False)
    root = tmp_path / "app"
    (root / "examples" / "mnist").mkdir(parents=True)
    net = root / "examples" / "mnist" / "lenet_train_test.prototxt"
    net.write_text("name: 'x'")
    model_dir = str(root / "examples" / "mnist")
    # placeholder resolved against the ancestors of the referring file
    assert paths.resolve("CAFFE_ROOT/examples/mnist/lenet_train_test.prototxt", model_dir) == str(net)
    # later lookups reuse the discovered root, also for files that do not exist (yet)
    assert paths.expand_placeholder("CAFFE_ROOT/examples/mnist/lenet", model_dir, must_exist=False) == \
        str(root / "examples" / "mnist" / "lenet")
    assert paths.resolve("CAFFE_ROOT/examples/mnist/mnist_train_lmdb", model_dir) == \
        str(root / "examples" / "mnist" / "mnist_train_lmdb")
    # repo-root-relative and model-dir-relative spellings
    assert paths.resolve("examples/mnist/lenet_train_test.prototxt", model_dir) == str(net)
    assert paths.resolve("lenet_train_test.prototxt", model_dir) == str(net)
    # a solver copied next to its net: stale directory part, found by file name (solver lookups only)
    assert paths.resolve("CAFFE_ROOT/old/place/lenet_train_test.prototxt", model_dir, basename_fallback=True) == str(net)
    assert paths.resolve("missing/file.prototxt", model_dir) == "missing/file.prototxt"
    # the environment variable wins
    monkeypatch.setenv("CAFFE_ROOT", "/opt/app")
    assert paths.resolve("CAFFE_ROOT/a/b", model_dir, must_exist=False) == "/opt/app/a/b"
    # models/bvlc_* of the reference use POSEIDON_ROOT
    assert paths.resolve("POSEIDON_ROOT/examples/mnist/lenet_train_test.prototxt", model_dir) == str(net)


def test_reference_example_solvers_load_unmodified():
    """examples/mnist + examples/cifar10 solver files of the reference (CAFFE_ROOT placeholders included) build nets."""
    import os
    from poseidon_b200 import get_solver, proto as P
    golden =os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")   # the reference's prototxt files
    ref = os.path.join(golden, "examples")
    for rel in ("mnist/lenet_solver.prototxt", "cifar10/cifar10_quick_solver.prototxt"):
        sp = P.read_solver(os.path.join(ref, rel))
        sp.snapshot, sp.snapshot_after_train, sp.display, sp.test_interval, sp.max_iter = 0, False, 0, 0, 1
        sp.clear("test_iter")
        s = get_solver(sp, engine="torch", model_dir=os.path.dirname(os.path.join(ref, rel)))
        s.step(1)
        assert s.net.layer_names and float(s.last_loss) > 0
        s.close()
    # deploy / full-convolutional / feature-extraction nets of the examples directory
    import torch
    from poseidon_b200 import Net
    for rel, top, shape in (("imagenet/bvlc_caffenet_full_conv.prototxt", "prob", (1, 1000, 8, 8)),
                            ("cifar10/cifar10_quick.prototxt", "prob", (1, 10, 1, 1)),
                            ("cifar10/cifar10_full.prototxt", "prob", (1, 10, 1, 1)),
                            ("feature_extraction/imagenet_val.prototxt", "loss", ())):
        net = Net(P.read_net(os.path.join(ref, rel)), phase=P.TEST)
        with torch.no_grad():
            _, out = net.forward({n: torch.rand(*net.blob_shapes[n]) for n in net.input_names})
        assert tuple(out[top].shape) == shape, rel
        net.close()
    # models/: POSEIDON_ROOT placeholders in net:, source:, mean_file:, snapshot_prefix: (built, not stepped: batch 256)
    mref = os.path.join(golden, "models/bvlc_alexnet/solver.prototxt")
    s = get_solver(P.read_solver(mref), engine="torch", model_dir=os.path.dirname(mref))
    assert s.net.layer_by_name["fc8"].weight.shape == (1000, 4096)
    assert "POSEIDON_ROOT" not in s._snapshot_prefix.__func__(type("S", (), {"param": s.param, "model_dir": s.model_dir, "snapshot_dir": "/tmp"})())
    s.close()
    for mref, n_ip in ((os.path.join(golden, "models/bvlc_googlenet/quick_solver.prototxt"), 5),
                       (os.path.join(golden, "models/bvlc_reference_caffenet/solver.prototxt"), 3)):
        s = get_solver(P.read_solver(mref), engine="torch", model_dir=os.path.dirname(mref))
        assert sum(1 for l in s.net.layers if l.type_name == "INNER_PRODUCT") == n_ip and len(s.test_nets) == 1
        s.close()


def test_lint_is_clean():
    """`make lint`: every Python file compiles, no unused imports, bounded line lengths (scripts/lint.py)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "scripts", "lint.py")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout[-3000:]


def test_bench_harness_two_ranks_on_emulated_fused_backend():
    """bench.py's multi-rank control flow (torchrun env, max over ranks, wire counters, e2e leg) with the sm100 engine
    and the fused backend, kernels and peer memory emulated — numbers are meaningless, keys and plumbing are checked."""
    import json
    import os
    import socket
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ, POSEIDON_EMULATE="1", OMP_NUM_THREADS="2")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "bench.py"),
                          "--gpus", "2", "--steps", "2", "--warmup", "3", "--allow-cpu", "--model", "lenet"],
                         capture_output=True, text=True, timeout=600, cwd=root, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1                                              # rank 0 only
    d = json.loads(lines[0])
    assert d["n_gpus"] == 2 and d["config"]["global_batch"] == 128 and d["config"]["parallelism"].startswith("dp2+dwbp")
    assert d["config"]["engine"] == "sm100" and d["config"]["comm"] == "fused"
    assert d["config"]["wire_bytes_total"]["dense_allreduce_bytes"] > 0 and d["gpu_launches"] > 0
    assert d["e2e"]["value"] > 0 and d["e2e"]["d2h_bytes_per_step"] == 4
    assert "resource_tracker" not in out.stderr


def test_hostfile_node_layout(tmp_path, monkeypatch):
    """Hostfile mode derives LOCAL_WORLD_SIZE / LOCAL_RANK (the per-node NVLink groups) from runs of equal hosts."""
    import os
    import pytest
    from poseidon_b200.parallel import context
    monkeypatch.setattr(context.dist, "init_process_group", lambda **kw: None)
    monkeypatch.setattr(context.dist, "is_initialized", lambda: False)
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT"):
        monkeypatch.delenv(k, raising=False)
    hf = tmp_path / "hosts"
    hf.write_text("0 10.0.0.1 9000\n1 10.0.0.1 9001\n2 10.0.0.2 9000\n3 10.0.0.2 9001\n")
    rc = context.init_rank_context("cpu", str(hf), client_id=3)
    assert (rc.rank, rc.world_size, rc.local_rank) == (3, 4, 1)
    assert os.environ["LOCAL_WORLD_SIZE"] == "2" and os.environ["LOCAL_RANK"] == "1" and os.environ["MASTER_ADDR"] == "10.0.0.1"
    for k in ("LOCAL_RANK", "LOCAL_WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT"):
        monkeypatch.delenv(k, raising=False)
    hf.write_text("0 10.0.0.1 9000\n1 10.0.0.2 9000\n2 10.0.0.1 9001\n3 10.0.0.2 9001\n")       # interleaved hosts
    with pytest.raises(ValueError, match="consecutive lines"):
        context.init_rank_context("cpu", str(hf), client_id=0)


def test_numa_affinity_policies(monkeypatch):
    """utils/affinity.py (NumaMgr's role): cpulist parsing, the 'even' slice per local rank, and 'center' degrading to
    the current CPU set when the GPU's NUMA node is unknown; the process affinity is restored afterwards."""
    import os
    from poseidon_b200.utils import affinity
    assert affinity._parse_cpulist("0-3,8,10-11") == [0, 1, 2, 3, 8, 10, 11]
    assert affinity.gpu_numa_node("ffff:ff:00.0") is None
    before = sorted(os.sched_getaffinity(0))
    try:
        assert affinity.pin_to_gpu_numa(0, "center") == before          # no GPU here: unchanged
        if len(before) >= 2:
            a = affinity.pin_to_gpu_numa(0, "even", local_rank=0, local_world=2)
            os.sched_setaffinity(0, before)
            b = affinity.pin_to_gpu_numa(0, "even", local_rank=1, local_world=2)
            assert a and b and not set(a) & set(b) and set(a) | set(b) <= set(before)
    finally:
        os.sched_setaffinity(0, before)
    assert sorted(os.sched_getaffinity(0)) == before
