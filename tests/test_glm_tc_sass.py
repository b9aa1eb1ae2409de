"""What ptxas makes of the wgmma GLM kernel (glm_tc.cu), checked without a GPU.

Both contractions of a tile are meant to run as one uninterrupted chain of wgmma instructions each.  ptxas
quietly serialises every wgmma of a kernel (a wait after each HGMMA) when ordinary instructions write an
accumulator inside a wgmma pipeline stage (note C7515) or when accumulators are live across a divergent
branch (C7520); the kernel still computes the right result, about 3x slower.  This test compiles glm_tc.cu
for sm_90a and checks, for both instantiations, that no such note is printed, that nothing spills, and that
no warpgroup wait or arrive sits between two HGMMA of the same contraction."""
import os
import re
import shutil
import subprocess

import pytest

from pyro_b200 import _build

KERNELS = {"default": "glm_bernoulli_tc_kernelILb0E", "split_x": "glm_bernoulli_tc_kernelILb1E"}


def _tools():
    try:
        nvcc = _build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    return nvcc, cuobjdump


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp("glm_tc_sass") / "glm_tc.o")
    src = os.path.join(_build.CSRC, "glm_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _ptxas_properties(log, mangled):
    """The 'N bytes stack frame, N bytes spill stores, N bytes spill loads' line and the register count."""
    lines = log.splitlines()
    for i, line in enumerate(lines):
        if "Function properties for" in line and mangled in line:
            props = lines[i + 1]
            used = next(l for l in lines[i + 1:] if "Used" in l and "registers" in l)
            return props, used
    raise AssertionError("ptxas printed no properties for %s:\n%s" % (mangled, log))


def _sass_function(sass, mangled):
    parts = re.split(r"^\s*Function : ", sass, flags=re.M)
    body = [p for p in parts if p.startswith("_Z") and mangled in p.split("\n", 1)[0]]
    assert len(body) == 1, "no SASS for %s" % mangled
    return [l for l in body[0].splitlines() if re.search(r"/\*[0-9a-f]{4,}\*/", l)]


@pytest.mark.parametrize("which", sorted(KERNELS))
def test_no_serialisation_note(compiled, which):
    log, _ = compiled
    for line in log.splitlines():
        if KERNELS[which] in line:
            assert "C7515" not in line and "C7520" not in line, line


@pytest.mark.parametrize("which", sorted(KERNELS))
def test_no_spills(compiled, which):
    log, _ = compiled
    props, used = _ptxas_properties(log, KERNELS[which])
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used


@pytest.mark.parametrize("which", sorted(KERNELS))
def test_one_wait_per_contraction(compiled, which):
    """Consecutive HGMMA of one shape form one contraction (GEMM 1 is m64n64k8, GEMM 2 m64n40k8); a
    WARPGROUP.DEPBAR or WARPGROUP.ARRIVE between two of them means ptxas broke the chain."""
    _, sass = compiled
    shapes, bad = [], []
    prev, between = None, []
    for line in _sass_function(sass, KERNELS[which]):
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            if m.group(1) == prev and between:
                bad.append("%s after %s" % (m.group(1), between))
            shapes.append(m.group(1))
            prev, between = m.group(1), []
        elif "WARPGROUP.DEPBAR" in line or "WARPGROUP.ARRIVE" in line:
            between.append(line.split(";")[0].split("*/")[-1].strip())
    assert "64x64x8" in shapes and "64x40x8" in shapes, shapes
    assert not bad, bad
