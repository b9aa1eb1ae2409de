"""Work per tile of the wgmma logistic-regression kernel (glm_tc.cu), checked in its SASS without a GPU.

The tile loop is limited by how long each warp's chain of instructions and MUFU ops is, so two savings are
pinned here for both instantiations: the epilogue takes one lg2 per particle and tile (of the product of the
softplus denominators) instead of one per logit, and the split pass writes X^T with 16-byte stores after a
register transpose instead of one 4-byte store per element.  The softmax kernel (glm_categorical_tc.cu) runs
the same D = 32 tile pipeline, so its split pass is held to the same stores."""
import re
import subprocess

import pytest

from pyro_b200 import _build
from test_glm_tc_sass import KERNELS, _sass_function, _tools

# the softmax kernel's instantiations (class padding x split X): mangled-name fragment -> split X
CATEGORICAL = {"glm_categorical_tc_kernelILi%dELb%dE" % (kp, sx): bool(sx) for kp in (2, 4, 8, 16) for sx in (0, 1)}


def _compile(tmp_path_factory, name):
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp("glm_tc_budget") / (name + ".o"))
    src = _build.CSRC + "/" + name + ".cu"
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-c", src, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    return _compile(tmp_path_factory, "glm_tc")


@pytest.fixture(scope="module")
def sass_categorical(tmp_path_factory):
    return _compile(tmp_path_factory, "glm_categorical_tc")


def _addr(line):
    return int(re.search(r"/\*([0-9a-f]{4,})\*/", line).group(1), 16)


def _tile_loop(lines):
    """The instructions of the tile loop: the widest backward branch whose body holds both contractions."""
    best = None
    for i, line in enumerate(lines):
        m = re.search(r"\bBRA(?:\.\S+)?\s+(?:\S+,\s*)?0x([0-9a-f]+)", line)
        if not m:
            continue
        target = int(m.group(1), 16)
        if target >= _addr(line):
            continue
        body = [l for l in lines[:i + 1] if _addr(l) >= target]
        text = "\n".join(body)
        if "HGMMA.64x64x8" in text and "HGMMA.64x40x8" in text and (best is None or len(body) > len(best)):
            best = body
    assert best is not None, "no backward branch encloses both contractions"
    return best


def _opcode(line):
    ins = line.split("*/", 1)[1].split(";")[0].strip()
    ins = re.sub(r"^@!?U?P\w+\s+", "", ins)
    return ins.split()[0] if ins else ""


@pytest.mark.parametrize("which", sorted(KERNELS))
def test_one_lg2_per_particle_and_tile(sass, which):
    loop = _tile_loop(_sass_function(sass, KERNELS[which]))
    ops = [_opcode(l) for l in loop]
    assert ops.count("MUFU.EX2") >= 32, ops.count("MUFU.EX2")
    assert ops.count("MUFU.LG2") <= 2, ops.count("MUFU.LG2")


@pytest.mark.parametrize("which", sorted(KERNELS) + sorted(CATEGORICAL))
def test_xt_written_with_vector_stores(sass, sass_categorical, which):
    """The only shared-memory stores in the tile loop are 16-byte ones: rounded X (and X_lo) in place and
    the rows of X^T."""
    if which in KERNELS:
        loop = _tile_loop(_sass_function(sass, KERNELS[which]))
        split_x = which == "split_x"
    else:
        loop = _tile_loop(_sass_function(sass_categorical, which))
        split_x = CATEGORICAL[which]
    ops = [_opcode(l) for l in loop]
    scalar = [op for op in ops if op.startswith("STS") and not op.startswith("STS.128")]
    assert not scalar, scalar
    assert ops.count("STS.128") == (12 if split_x else 8), ops.count("STS.128")
