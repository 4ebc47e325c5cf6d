"""CPU-side checks of the code ptxas makes of the TMA-staged convolution kernel (conv_tma.cu): every instance keeps its
wgmma instructions pipelined (no arrive injected by the compiler, no serialisation), spills nothing, and issues one
full-width m64 x BN x k16 instruction per product and K step."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "conv_tma_kernel"
# conv_tma_kernel<kNPass, kBN, kBf16>, as mangled: ..._kernelILi3ELi128ELb0EE...
INSTANCE = re.compile(r"conv_tma_kernelILi(\d+)ELi(\d+)ELb([01])E")
EXPECTED = {(p, bn, bf) for p in (1, 3) for bn in (32, 64, 96, 128) for bf in (0, 1)}


def _nvcc():
    return os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    from coclr_b200 import build
    out = tmp_path_factory.mktemp("conv_tma_sass")
    cmd = [_nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "conv_tma.cu"),
                                          "-o", str(out / "conv_tma.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


def test_every_instance_is_compiled(ptxas_log):
    found = {(int(p), int(bn), int(bf)) for p, bn, bf in INSTANCE.findall(ptxas_log)}
    assert found == EXPECTED, found ^ EXPECTED


def test_wgmma_is_not_serialised_or_patched_by_ptxas(ptxas_log):
    bad = [l for l in ptxas_log.splitlines() if KERNEL in l and
           ("warpgroup.arrive is injected" in l or "are serialized" in l)]
    assert not bad, "\n".join(bad[:5])


def test_no_spills(ptxas_log):
    lines = ptxas_log.splitlines()
    checked = 0
    for i, l in enumerate(lines):
        if "Function properties for" in l and KERNEL in l:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            assert m, lines[i + 1]
            assert (int(m.group(1)), int(m.group(2))) == (0, 0), (l, lines[i + 1])
            checked += 1
    assert checked == len(EXPECTED), checked


def test_each_instance_issues_full_width_hgmma():
    from coclr_b200 import build
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", build.build()], capture_output=True, text=True).stdout
    bodies = re.split(r"\n\s*Function : ", sass)
    seen = set()
    for body in bodies:
        name = body.split("\n", 1)[0]
        m = INSTANCE.search(name)
        if not m:
            continue
        npass, bn, bf = int(m.group(1)), int(m.group(2)), int(m.group(3))
        seen.add((npass, bn, bf))
        widths = set(re.findall(r"HGMMA\.64x(\d+)x16", body))
        assert widths == {str(bn)}, (name, widths)
    assert seen == EXPECTED, seen ^ EXPECTED
