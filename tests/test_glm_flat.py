"""The logistic-regression likelihood on the tensor cores for every feature count D in 1..128 that has no
kernel of its own (glm_flat_tc.cu): each 64-row tile of X arrives by one 1-D bulk copy into a [64][D]
landing buffer, and the split pass pads D to whole 32-column swizzle atoms.

CPU tier: what ptxas makes of every instantiation (no serialisation note, no spills, one wgmma chain per
contraction, at most 2 MUFU.LG2 in the tile loop) and the entry point's argument checks.
GPU tier: the kernel against fp64 at full size and at ragged shapes, the unchanged `logistic_model` at D = 10
and 100 against the oracle and the materialised path, graph capture, and the sites that keep the
materialised path."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

import models
import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from oracle import dists as od
from oracle import svi as osvi
from pyro_b200 import _build
from pyro_b200 import _native as N
from pyro_b200.infer import SVI, JitTrace_ELBO, Trace_ELBO
from pyro_b200.infer import elbo as elbo_mod
from pyro_b200.optim import ClippedAdam

DEV = device()
# (atoms of 32 columns, split X) -> mangled-name fragment
KERNELS = {(dc, sx): "glm_bernoulli_flat_tc_kernelILi%dELb%dE" % (dc, int(sx)) for dc in (1, 2, 3, 4)
           for sx in (False, True)}
IDS = ["DC%d-%s" % (dc, "split_x" if sx else "default") for dc, sx in sorted(KERNELS)]


# ---- CPU tier: SASS ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    from test_glm_tc_sass import _tools
    nvcc, cuobjdump = _tools()
    obj = str(tmp_path_factory.mktemp("glm_flat_sass") / "glm_flat_tc.o")
    src = os.path.join(_build.CSRC, "glm_flat_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _addr(line):
    return int(re.search(r"/\*([0-9a-f]{4,})\*/", line).group(1), 16)


def _opcode(line):
    ins = line.split("*/", 1)[1].split(";")[0].strip()
    ins = re.sub(r"^@!?U?P\w+\s+", "", ins)
    return ins.split()[0] if ins else ""


def _tile_loop(lines, g2):
    """The instructions of the tile loop: the widest backward branch whose body holds both contractions."""
    best = None
    for i, line in enumerate(lines):
        m = re.search(r"\bBRA(?:\.\S+)?\s+(?:\S+,\s*)?0x([0-9a-f]+)", line)
        if not m or int(m.group(1), 16) >= _addr(line):
            continue
        body = [l for l in lines[:i + 1] if _addr(l) >= int(m.group(1), 16)]
        text = "\n".join(body)
        if "HGMMA.64x64x8" in text and "HGMMA.%s" % g2 in text and (best is None or len(body) > len(best)):
            best = body
    assert best is not None, "no backward branch encloses both contractions"
    return best


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_no_serialisation_note_and_no_spills(compiled, key):
    from test_glm_tc_sass import _ptxas_properties
    log, _ = compiled
    assert "C7515" not in log and "C7520" not in log, log
    props, used = _ptxas_properties(log, KERNELS[key])
    assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", props), props + " / " + used


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_one_wait_per_contraction(compiled, key):
    """GEMM 1 is m64n64k8 over 4 DC k-steps (2 or 3 split products each), GEMM 2 m64n(32 DC + 8)k8 over 8
    k-steps; a WARPGROUP.DEPBAR or WARPGROUP.ARRIVE between two HGMMA of one shape breaks the chain."""
    from test_glm_tc_sass import _sass_function
    dc, split_x = key
    g2 = "64x%dx8" % (32 * dc + 8)
    _, sass = compiled
    shapes, bad = [], []
    prev, between = None, []
    for line in _sass_function(sass, KERNELS[key]):
        m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
        if m:
            if m.group(1) == prev and between:
                bad.append("%s after %s" % (m.group(1), between))
            shapes.append(m.group(1))
            prev, between = m.group(1), []
        elif "WARPGROUP.DEPBAR" in line or "WARPGROUP.ARRIVE" in line:
            between.append(line.split(";")[0].split("*/")[-1].strip())
    assert shapes.count("64x64x8") == 4 * dc * (3 if split_x else 2), shapes
    assert shapes.count(g2) == 8, shapes
    assert not bad, bad


@pytest.mark.parametrize("key", sorted(KERNELS), ids=IDS)
def test_one_lg2_per_particle_and_tile(compiled, key):
    from test_glm_tc_sass import _sass_function
    _, sass = compiled
    loop = _tile_loop(_sass_function(sass, KERNELS[key]), "64x%dx8" % (32 * key[0] + 8))
    ops = [_opcode(l) for l in loop]
    assert ops.count("MUFU.EX2") >= 32, ops.count("MUFU.EX2")
    assert ops.count("MUFU.LG2") <= 2, ops.count("MUFU.LG2")


# ---- CPU tier: argument checks -----------------------------------------------------------------------------
def test_entry_point_validates_feature_count_before_any_cuda_call():
    """D outside 1..128, and the fp32 SIMT flag with a D the SIMT kernel lacks, are refused with
    B2_ERR_BAD_SHAPE; so is a y that is not 16-byte aligned at such a D.  The pointers are never
    dereferenced and no workspace is passed: the shape checks come first."""
    L = N.lib()
    assert L.b2_version() >= 104
    p = ctypes.c_void_p(4096)
    q = ctypes.c_void_p(4100)

    def call(X, y, n, D, flags):
        return L.b2_glm_bernoulli_logits(X, y, p, None, n, D, 8, 1.0, 1.0, 1.0, flags, None, None, None, None,
                                         None, 0, None)

    assert call(p, p, 10000, 0, 0) == -2
    assert call(p, p, 10000, 129, 0) == -2
    assert call(p, p, 10000, -3, 0) == -2
    assert call(p, p, 10000, 10, N.B2_FLAG_GLM_FP32) == -2
    assert call(p, q, 10000, 10, 0) == -2                     # y not 16-byte aligned
    assert call(p, p, 1 << 31, 10, 0) == -8                   # 32-bit row counts
    # a valid shape reaches the workspace check; so do the D that keep their own kernels
    for D in (1, 10, 33, 128):
        assert call(p, p, 10000, D, 0) == -5, D
    assert call(p, q, 10000, 32, N.B2_FLAG_GLM_FP32) == -5


# ---- GPU tier: the kernel against fp64 ---------------------------------------------------------------------
def _launch(X, y, W, b, flags):
    n, D = X.shape
    P = W.shape[0]
    sum_p = torch.empty(P, device=DEV)
    total = torch.empty((), device=DEV)
    dW = torch.empty(P, D, device=DEV)
    db = torch.empty(P, device=DEV)
    ws = N.workspace(torch.device(DEV), int(N.lib().b2_glm_workspace(n, D, P)), tag="glm_flat")
    N.check(N.lib().b2_glm_bernoulli_logits(X.data_ptr(), y.data_ptr(), W.data_ptr(),
                                            b.data_ptr() if b is not None else None, n, D, P, 1.0, 1.0, 1.0,
                                            flags, sum_p.data_ptr(), total.data_ptr(), dW.data_ptr(),
                                            db.data_ptr(), ws.data_ptr(), ws.numel(),
                                            N.stream_ptr(torch.device(DEV))), "b2_glm_bernoulli_logits")
    torch.cuda.synchronize()
    return sum_p, total, dW, db


def _reference(X, y, W, b):
    """fp64 per-particle sums and their gradients by autograd through oracle/dists.py (on the device)."""
    Wd = W.double().requires_grad_(True)
    bd = (b if b is not None else torch.zeros(W.shape[0], device=W.device)).double().requires_grad_(True)
    s = od.bernoulli_logits(y.double(), Wd @ X.double().t() + bd[:, None]).sum(1)
    gW, gb = torch.autograd.grad(s.sum(), [Wd, bd])
    return s.detach(), gW, gb


_FULL = {}


@pytest.mark.gpu
@pytest.mark.parametrize("flag_name", ["default", "B2_FLAG_GLM_3XTF32"])
@pytest.mark.parametrize("D", [1, 10, 33, 54, 64, 100, 127, 128])
def test_flat_kernel_full_size_against_oracle(D, flag_name):
    """N = 1e6, P = 64: sums within 2e-5 relative, dW and db within 2e-4 of the largest gradient (the
    tolerances of the D = 32 kernel), and two launches are bitwise equal."""
    if EMULATE:
        pytest.skip("kernel test")
    n, P = 1_000_000, 64
    if D not in _FULL:
        _FULL.clear()
        g = torch.Generator().manual_seed(100 + D)
        X = torch.randn(n, D, generator=g)
        wt = torch.randn(D, generator=g) / D ** 0.5
        y = (torch.rand(n, generator=g) < torch.sigmoid(X @ wt + 0.5)).float()
        W = 0.3 * torch.randn(P, D, generator=g) / D ** 0.5 + wt
        b = 0.5 + 0.2 * torch.randn(P, generator=g)
        Xg, yg, Wg, bg = X.to(DEV), y.to(DEV), W.to(DEV), b.to(DEV)
        _FULL[D] = (Xg, yg, Wg, bg) + _reference(Xg, yg, Wg, bg)
    Xg, yg, Wg, bg, s_ref, gW, gb = _FULL[D]
    flags = 0 if flag_name == "default" else getattr(N, flag_name)
    sum_p, total, dW, db = _launch(Xg, yg, Wg, bg, flags)
    assert float(((sum_p.double() - s_ref).abs() / s_ref.abs()).max()) <= 2e-5
    assert abs(float(total) - float(s_ref.sum())) <= 2e-5 * abs(float(s_ref.sum()))
    assert float((dW.double() - gW).abs().max()) <= 2e-4 * float(gW.abs().max())
    assert float((db.double() - gb).abs().max()) <= 2e-4 * float(gb.abs().max())
    sum2, total2, dW2, db2 = _launch(Xg, yg, Wg, bg, flags)
    assert torch.equal(sum_p, sum2) and torch.equal(total, total2)
    assert torch.equal(dW, dW2) and torch.equal(db, db2)


# (n, P, D, bias, flag): every n, P and D of the ragged set, with and without a bias; the last tile of
# 70001 rows holds 49 rows, so at odd D its byte count is not a multiple of 16; n = 1 and 63 at P = 1 are a
# CTA's only, partial tile and the first use of its buffers
_RAGGED = [(1, 1, 1, True, None), (1, 1, 33, False, "B2_FLAG_GLM_3XTF32"), (63, 1, 3, True, None),
           (63, 1, 127, False, None), (64, 3, 10, False, None), (65, 65, 33, True, None),
           (65, 130, 1, False, "B2_FLAG_GLM_3XTF32"), (8192, 64, 127, True, None), (8192, 3, 3, False, None),
           (65535, 130, 10, True, None), (65535, 65, 127, False, None), (70001, 64, 3, True, None),
           (70001, 65, 33, False, None), (70001, 130, 127, True, "B2_FLAG_GLM_3XTF32"), (70001, 1, 1, False, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,P,D,bias,flag", _RAGGED, ids=["-".join(map(str, c)) for c in _RAGGED])
def test_flat_kernel_ragged_shapes_against_oracle(n, P, D, bias, flag):
    """Tolerances of the D = 32 ragged test: 2e-5 on the sums; on the gradients 2e-4 from 8192 rows and 5e-4
    below, where the single-pass TF32 gradient contraction has nothing to average over (these D have no
    fp32 kernel to fall back to)."""
    if EMULATE:
        pytest.skip("kernel test")
    g = torch.Generator().manual_seed(7 * n + 3 * P + D)
    X = torch.randn(n, D, generator=g)
    y = (torch.rand(n, generator=g) < 0.4).float()
    W = 0.3 * torch.randn(P, D, generator=g)
    b = torch.randn(P, generator=g) if bias else None
    Xg, yg, Wg = X.to(DEV), y.to(DEV), W.to(DEV)
    bg = b.to(DEV) if bias else None
    s_ref, gW, gb = _reference(Xg, yg, Wg, bg)
    sum_p, total, dW, db = _launch(Xg, yg, Wg, bg, getattr(N, flag) if flag else 0)
    tol_g = 2e-4 if n >= 8192 else 5e-4
    assert float((sum_p.double() - s_ref).abs().max()) <= 2e-5 * max(1.0, float(s_ref.abs().max()))
    assert float((dW.double() - gW).abs().max()) <= tol_g * max(1.0, float(gW.abs().max()))
    if bias:
        assert float((db.double() - gb).abs().max()) <= tol_g * max(1.0, float(gb.abs().max()))


# ---- GPU tier: the unchanged model -------------------------------------------------------------------------
def _noise(eps_w, eps_b, box):
    def guide(X_, y_):
        with models.InjectNoise({"w": eps_w[box["i"]], "b": eps_b[box["i"]]}):
            models.logistic_guide(X_, y_)
    return guide


def _run(model, X, y, eps_w, eps_b, lazy, elbo_cls=Trace_ELBO, extra=()):
    """Steps of SVI on `model` with noise injected through fixed device buffers, so eager and captured runs
    consume identical draws; returns the losses, the parameters and the number of kernel calls."""
    pyro.clear_param_store()
    bw, bb = torch.empty_like(eps_w[0]), torch.empty_like(eps_b[0])
    box = {"i": 0}
    calls = []
    real = dist._GlmBernoulliFn.apply

    def spy(*a):
        calls.append(1)
        return real(*a)

    def guide(*args):
        with models.InjectNoise({"w": bw, "b": bb}):
            models.logistic_guide(*args[:2])

    saved = elbo_mod.LAZY_LINEAR
    elbo_mod.LAZY_LINEAR = lazy
    dist._GlmBernoulliFn.apply = spy
    try:
        svi = SVI(model, guide, ClippedAdam({"lr": 0.01}),
                  elbo_cls(num_particles=eps_w.shape[1], vectorize_particles=True, max_plate_nesting=1))
        losses = []
        for i in range(eps_w.shape[0]):
            bw.copy_(eps_w[i])
            bb.copy_(eps_b[i])
            losses.append(svi.step(X, y, *extra))
    finally:
        elbo_mod.LAZY_LINEAR = saved
        dist._GlmBernoulliFn.apply = real
    store = pyro.get_param_store()
    return losses, {k: store[k].detach().clone() for k in ("w_loc", "w_scale", "b_loc", "b_scale")}, len(calls)


def _data(n, D, P, steps, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, D, generator=g, dtype=torch.float64)
    y = (torch.rand(n, generator=g, dtype=torch.float64) < torch.sigmoid(X[:, 0] - 0.5 * X[:, 1] + 0.25)).double()
    eps_w = torch.randn(steps, P, 1, D, generator=g, dtype=torch.float64)
    eps_b = torch.randn(steps, P, 1, generator=g, dtype=torch.float64)
    return X.to(dtype), y.to(dtype), eps_w.to(dtype), eps_b.to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 100])
def test_unchanged_logistic_model_matches_oracle_and_materialised(D):
    """`models.logistic_model` (the reference model verbatim) at N = 70 000, P = 16: every step's likelihood
    site is scored by the kernel, and three SVI steps match oracle/svi.py with the tolerances of the D = 32
    test (loss 2e-5 relative, parameters 2e-4) and the materialised path (LAZY_LINEAR = False)."""
    if EMULATE:
        pytest.skip("kernel test")
    n, P = 70000, 16
    X, y, eps_w, eps_b = _data(n, D, P, 3, D)
    ref = osvi.LogisticSVIMatmul(D, P, lr=0.01)
    ref_losses = [ref.step(X, y, eps_w[i], eps_b[i]) for i in range(3)]
    Xd, yd, ew, eb = X.to(DEV), y.to(DEV), eps_w.to(DEV), eps_b.to(DEV)
    seen = []
    real = dist._BernoulliLinear._fused_sum

    def spy(self, *a, **k):
        seen.append(type(self).__name__)
        return real(self, *a, **k)
    dist._BernoulliLinear._fused_sum = spy
    try:
        l_f, p_f, calls = _run(models.logistic_model, Xd, yd, ew, eb, True)
    finally:
        dist._BernoulliLinear._fused_sum = real
    assert len(seen) == 3 and calls == 3
    for i in range(3):
        assert abs(l_f[i] - ref_losses[i]) <= 2e-5 * abs(ref_losses[i]), (i, l_f[i], ref_losses[i])
    cons = ref.constrained()
    for k in p_f:
        assert torch.allclose(p_f[k].cpu().reshape(-1), cons[k].reshape(-1), atol=2e-4), k
    l_m, p_m, calls_m = _run(models.logistic_model, Xd, yd, ew, eb, False)
    assert calls_m == 0
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= 2e-5 * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=2e-4), k


@pytest.mark.gpu
def test_captured_graph_step_equals_eager_d100():
    """JitTrace_ELBO (the step captured in a CUDA graph) gives bit for bit the losses and parameters of the
    eager steps at D = 100, with every scoring of the site, the capturing one included, on the kernel."""
    if EMULATE:
        pytest.skip("graph capture needs a GPU")
    X, y, eps_w, eps_b = _data(70000, 100, 16, 4, 5)
    X, y, eps_w, eps_b = X.to(DEV), y.to(DEV), eps_w.to(DEV), eps_b.to(DEV)
    l_e, p_e, n_e = _run(models.logistic_model, X, y, eps_w, eps_b, True)
    l_g, p_g, n_g = _run(models.logistic_model, X, y, eps_w, eps_b, True, JitTrace_ELBO)
    assert n_e == 4 and n_g >= 3
    assert l_e == l_g, (l_e, l_g)
    for k in p_e:
        assert torch.equal(p_e[k], p_g[k]), k


def logistic_model_masked(X, y, mask):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=w.squeeze(-2) @ X.T + b).mask(mask), obs=y)


def logistic_model_simt(X, y):
    """A lazy predictor that asks for the fp32 SIMT contractions (tensor_cores=False)."""
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=dist.linear_predictor(X, w, b, tensor_cores=False)), obs=y)


def logistic_model_simt_eager(X, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), X.new_ones(D)).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), X.new_full((), 10.0)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=w.squeeze(-2) @ X.T + b), obs=y)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["D129", "N8191", "masked", "fp64", "y_offset1", "no_tensor_cores"])
def test_out_of_scope_sites_keep_the_materialised_path(case):
    """Sites outside the kernel's scope make no kernel call and give the results of LAZY_LINEAR = False:
    D = 129, N = 8191, a masked site, fp64, a y that is not 16-byte aligned, and tensor_cores=False."""
    if EMULATE:
        pytest.skip("kernel test")
    n, D, P = 9000, 10, 4
    dtype = torch.float64 if case == "fp64" else torch.float32
    if case == "D129":
        D = 129
    if case == "N8191":
        n = 8191
    X, y, eps_w, eps_b = _data(n, D, P, 2, 31, dtype)
    X, y, eps_w, eps_b = X.to(DEV), y.to(DEV), eps_w.to(DEV), eps_b.to(DEV)
    model, model_m, extra = models.logistic_model, models.logistic_model, ()
    if case == "masked":
        model = model_m = logistic_model_masked
        extra = (torch.rand(n, device=DEV) < 0.7,)
    if case == "y_offset1":
        y = torch.cat([torch.zeros(1, device=DEV), y])[1:]
        assert y.data_ptr() % 16 != 0
    if case == "no_tensor_cores":
        model, model_m = logistic_model_simt, logistic_model_simt_eager
    l_f, p_f, calls = _run(model, X, y, eps_w, eps_b, True, extra=extra)
    assert calls == 0
    l_m, p_m, _ = _run(model_m, X, y, eps_w, eps_b, False, extra=extra)
    tol = 1e-12 if dtype == torch.float64 else 2e-6
    for a, b in zip(l_f, l_m):
        assert abs(a - b) <= tol * abs(b), (l_f, l_m)
    for k in p_m:
        assert torch.allclose(p_f[k], p_m[k], atol=tol, rtol=tol), k
