"""The in-tree extension really is Hopper-native: `cuobjdump -sass` of the built .so (no GPU needed) must show the
wgmma / TMA / multimem instruction families in the kernels that claim them — and no legacy `mma.sync` (HMMA) anywhere.
    wgmma.mma_async -> HGMMA, TMA tile / im2col loads -> UTMALDG (.IM2COL, .MULTICAST for cluster-shared tiles),
    bulk async stores -> UBLKCP, multimem.ld_reduce -> LDGMC.E.ADD (multimem.st is a system-scope STG to the multicast address)."""
import os
import re
import shutil
import subprocess

import pytest

SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "poseidon_b200", "_ext", "poseidon_b200_C.so")


@pytest.fixture(scope="module")
def sass():
    if not os.path.exists(SO) or shutil.which("cuobjdump") is None:
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, timeout=600).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and "/*" in line and ";" in line:
            funcs[cur].append(line)
    assert len(funcs) > 100, len(funcs)
    return {k: "\n".join(v) for k, v in funcs.items()}


def _kernels(sass, needle):
    return {k: v for k, v in sass.items() if needle in k}


def test_gemm_core_uses_wgmma_and_tma(sass):
    gemm = _kernels(sass, "wgmma_gemm_kernel")
    assert len(gemm) >= 40, len(gemm)
    for name, text in gemm.items():
        assert re.search(r"HGMMA\.64x\d+x16\.F32\.BF16", text), f"no wgmma in {name}"
        assert "UTMALDG" in text, f"no TMA load in {name}"
        assert not re.search(r"\bHMMA", text), f"legacy mma.sync in {name}"
    assert any("HGMMA.64x256x16" in t for t in gemm.values()), "no 256-wide wgmma tile"
    assert any("UTMALDG.2D.MULTICAST" in t for t in gemm.values()), "no CTA-pair multicast of the B tile"
    assert any(re.search(r"UTMALDG\.\dD\.IM2COL", t) for t in gemm.values()), "no im2col-mode TMA"
    assert any("UTMALDG.4D.IM2COL.MULTICAST" in t for t in gemm.values()), "no cluster-shared im2col loads"
    assert any("UBLKCP" in t for t in gemm.values()), "no bulk-async row stores in any epilogue"


def test_comm_kernels_use_multimem(sass):
    ar = _kernels(sass, "allreduce_sgd")
    assert ar, "all-reduce + SGD kernels missing"
    assert any(re.search(r"LDGMC\.E\.ADD\.F32x4", t) for t in ar.values()), "no multimem.ld_reduce (in-switch fp32 add)"
    # multimem.st has no mnemonic of its own: ptxas emits a system-scope STG to the multicast address
    assert any(re.search(r"STG\.E\.128\.STRONG\.SYS", t) for t in ar.values()), "no 16-byte system-scope store"


def test_no_legacy_tensor_core_path_anywhere(sass):
    offenders = [k for k, t in sass.items() if re.search(r"\bHMMA", t)]
    assert not offenders, offenders[:3]
