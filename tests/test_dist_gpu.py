"""Multi-GPU (>= 2 H100) checks of the fused NVLink backend: in-kernel all-reduce + optimizer, fused SFB,
against single-GPU training on the concatenated batch; plus the NCCL baseline."""
import numpy as np
import pytest

from test_dist_cpu import _weights, launch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def _close(a, b, rel, floor=2e-4):
    for k in _weights(a):
        d = np.abs(a[k] - b[k]).max()
        m = np.abs(b[k]).max() + 1e-6
        assert d <= rel * m + floor, (k, d, m)


@pytest.fixture(scope="module")
def single_sm100(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("single_gpu") / "w")
    return launch(1, out, ["--batch", "16", "--base_lr", "0.02", "--engine", "sm100", "--hw", "35"], device=None)[0]


def test_fused_allreduce_sgd_two_ranks(tmp_path, single_sm100):
    res = launch(2, str(tmp_path / "w"), ["--batch", "8", "--engine", "sm100", "--comm", "fused", "--svb", "0",
                                            "--hw", "35"], device=None)
    _close(res[0], res[1], 1e-6)                     # replicas bit-close
    _close(res[0], single_sm100, 0.03)               # == one GPU on the concatenated batch (bf16 noise)
    assert int(res[0]["wire_dense_allreduce_bytes"]) > 0


def test_fused_sfb_two_ranks(tmp_path, single_sm100):
    res = launch(2, str(tmp_path / "w"), ["--batch", "8", "--engine", "sm100", "--comm", "fused", "--svb", "1",
                                            "--sfb_mode", "all", "--hw", "35"], device=None)
    _close(res[0], res[1], 1e-6)
    _close(res[0], single_sm100, 0.03)
    assert int(res[0]["wire_sfb_bytes"]) > 0


def test_nccl_baseline_two_ranks(tmp_path):
    ref = launch(1, str(tmp_path / "s"), ["--batch", "16", "--base_lr", "0.02", "--hw", "35"], device=None)[0]
    res = launch(2, str(tmp_path / "w"), ["--batch", "8", "--comm", "nccl", "--hw", "35"], device=None)
    _close(res[0], ref, 1e-3)


@pytest.mark.parametrize("comm", [["--comm", "fused", "--svb", "1", "--sfb_mode", "all"], ["--comm", "nccl"],
                                  ["--comm", "ssp", "--staleness", "1"]])
def test_two_gpu_snapshot_and_resume(tmp_path, monkeypatch, comm):
    """The CPU-emulated test_multi_rank_snapshot_and_resume_is_exact on real kernels / NVLink / NCCL: 2 steps + snapshot
    (sharded history gathered by every rank), restore in a fresh job, 2 more steps == 4 uninterrupted steps.  The SSP
    case also re-runs the NCCL wire-buffer path that failed once at 8 GPUs."""
    monkeypatch.setenv("POSEIDON_ONE_SHOT_BYTES", "1024")
    base = ["--batch", "8", "--engine", "sm100", "--hw", "35"] + comm
    full = launch(2, str(tmp_path / "A"), base + ["--steps", "4"], device=None)
    launch(2, str(tmp_path / "B"), base + ["--steps", "2", "--total_steps", "4", "--snapshot_prefix",
                                            str(tmp_path / "snap")], device=None)
    state = str(tmp_path / "snap_iter_2.solverstate")
    res = launch(2, str(tmp_path / "C"), base + ["--steps", "2", "--total_steps", "4", "--restore", state], device=None)
    _close(res[0], res[1], 1e-6 if comm[1] != "ssp" else 0.05)
    _close(res[0], full[0], 0.02 if comm[1] != "ssp" else 0.2)


def test_fused_ssp_two_ranks_staleness_zero_matches_library_ssp(tmp_path, monkeypatch):
    """The SSP kernels on the NVLink arena (ssp_delta / ssp_fold: per-worker deltas in a ring, folded by the peers over
    P2P loads, no NCCL on the path) at staleness 0 = BSP with summed per-worker updates = the library SSP backend."""
    monkeypatch.setenv("POSEIDON_FUSED_SSP", "1")
    base = ["--batch", "8", "--engine", "sm100", "--hw", "35"]
    res = launch(2, str(tmp_path / "f"), base + ["--comm", "fused", "--staleness", "0"], device=None)
    lib = launch(2, str(tmp_path / "l"), base + ["--comm", "ssp", "--staleness", "0"], device=None)
    _close(res[0], res[1], 1e-5)
    _close(res[0], lib[0], 0.03)
    assert int(res[0]["max_lag"]) == 0 and int(res[0]["wire_ssp_delta_bytes"]) > 0


@pytest.mark.parametrize("staleness", [1, 2])
def test_fused_ssp_straggler_stays_within_the_staleness_bound(tmp_path, monkeypatch, staleness):
    """An injected straggler (POSEIDON_FAULT delay on rank 1): no worker ever sees a peer more than `staleness` clocks
    behind, every delta is folded exactly once (replicas agree after the drain), training stays finite and near the
    library SSP trajectory."""
    monkeypatch.setenv("POSEIDON_FAULT", "delay:rank=1,step=2,ms=300")
    base = ["--batch", "8", "--engine", "sm100", "--hw", "35", "--steps", "6", "--staleness", str(staleness)]
    res = launch(2, str(tmp_path / "f"), base + ["--comm", "fused"], device=None)
    _close(res[0], res[1], 1e-4)
    assert all(int(r["max_lag"]) <= staleness for r in res)
    assert np.isfinite(res[0]["loss"])
    lib = launch(2, str(tmp_path / "l"), base + ["--comm", "ssp"], device=None)
    # two asynchronous runs whose fold order depends on timing: same neighbourhood, not the same trajectory (the
    # absolute floor covers the biases, which start at zero and are ~1e-2 after six steps)
    _close(res[0], lib[0], 0.3, floor=1e-3)


@pytest.mark.parametrize("graph", ["0", "1"], ids=["eager", "cuda_graph"])
def test_fused_branch_parallel_lanes_two_ranks(tmp_path, monkeypatch, graph):
    """A branchy net (two inception modules + an auxiliary head) on 2 GPUs with the layers of independent branches on
    separate streams: DWBP buckets are launched from hooks that fire on the lane streams, the fused all-reduce + SGD
    kernels wait on those — the replicas must stay bit-close and follow one GPU on the concatenated batch."""
    base = ["--engine", "sm100", "--net", "inception", "--steps", "4", "--graph", graph]
    monkeypatch.setenv("POSEIDON_LANES", "1")
    ref = launch(1, str(tmp_path / "s"), base + ["--batch", "16", "--base_lr", "0.02"], device=None)[0]
    monkeypatch.setenv("POSEIDON_LANES", "4")
    res = launch(2, str(tmp_path / "w"), base + ["--batch", "8", "--comm", "fused", "--svb", "1", "--sfb_mode", "all"],
                 device=None)
    _close(res[0], res[1], 1e-6)
    _close(res[0], ref, 0.03)
