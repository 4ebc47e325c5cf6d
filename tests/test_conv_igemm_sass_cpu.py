"""CPU-side checks of the code ptxas makes of the gather kernels of conv_igemm.cu (the convolution kernel
conv_igemm_kernel and the weight-gradient kernel conv_wgrad_kernel): every instance is compiled, keeps its wgmma
instructions pipelined (no arrive injected by the compiler, no serialisation), spills nothing, and issues only the
instruction width of its shape."""
import os
import re
import subprocess

import pytest

# kernel -> (mangled-instance regex, expected instances, HGMMA widths of an instance)
KERNELS = {
    # conv_igemm_kernel<kNPass, kBN, kBf16>, as mangled: ..._kernelILi3ELi128ELb0EE...; one full-width m64 x BN x k16
    # instruction per product and K step
    "conv_igemm_kernel": (re.compile(r"conv_igemm_kernelILi(\d+)ELi(\d+)ELb([01])E"),
                          {(p, bn, bf) for p in (1, 3) for bn in (32, 64, 96, 128) for bf in (0, 1)},
                          lambda npass, bn, bf: {str(bn)}),
    # conv_wgrad_kernel<kNProd, kBNk, kBf16>: one m64 x 64 x k16 instruction per 64-column block, product and K step
    "conv_wgrad_kernel": (re.compile(r"conv_wgrad_kernelILi(\d+)ELi(\d+)ELb([01])E"),
                          {(p, bnk, bf) for p in (1, 2, 3) for bnk in (64, 128) for bf in (0, 1)},
                          lambda nprod, bnk, bf: {"64"}),
}


def _nvcc():
    return os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    from coclr_b200 import build
    out = tmp_path_factory.mktemp("conv_igemm_sass")
    cmd = [_nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "conv_igemm.cu"),
                                          "-o", str(out / "conv_igemm.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


def test_every_instance_is_compiled(ptxas_log):
    for kernel, (instance, expected, _) in KERNELS.items():
        found = {tuple(int(v) for v in m) for m in instance.findall(ptxas_log)}
        assert found == expected, (kernel, found ^ expected)


def test_wgmma_is_not_serialised_or_patched_by_ptxas(ptxas_log):
    bad = [l for l in ptxas_log.splitlines() if any(k in l for k in KERNELS) and
           ("warpgroup.arrive is injected" in l or "are serialized" in l)]
    assert not bad, "\n".join(bad[:5])


def test_no_spills(ptxas_log):
    lines = ptxas_log.splitlines()
    for kernel, (_, expected, _) in KERNELS.items():
        checked = 0
        for i, l in enumerate(lines):
            if "Function properties for" in l and kernel in l:
                m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
                assert m, lines[i + 1]
                assert (int(m.group(1)), int(m.group(2))) == (0, 0), (l, lines[i + 1])
                checked += 1
        assert checked == len(expected), (kernel, checked)


def test_each_instance_issues_full_width_hgmma():
    from coclr_b200 import build
    cuobjdump = os.path.join(os.path.dirname(_nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", build.build()], capture_output=True, text=True).stdout
    bodies = re.split(r"\n\s*Function : ", sass)
    for kernel, (instance, expected, widths_of) in KERNELS.items():
        seen = set()
        for body in bodies:
            name = body.split("\n", 1)[0]
            m = instance.search(name)
            if not m:
                continue
            key = tuple(int(v) for v in m.groups())
            seen.add(key)
            widths = set(re.findall(r"HGMMA\.64x(\d+)x16", body))
            assert widths == widths_of(*key), (name, widths)
        assert seen == expected, (kernel, seen ^ expected)
