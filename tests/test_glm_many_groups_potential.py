"""GlmPotential past 128 columns: a group effect whose one-hot columns do not fit the contraction
(D + G (1 + S) > 128) is gathered per row and its gradient summed over each group's rows, which needs the rows sorted
by group.  Recognition and layout against TracePotential, the near misses that keep TracePotential, the C ABI's checks
and the new kernels' SASS (CPU tier); U and dU/dz against fp64 and TracePotential, ragged layouts, the NaN policy,
graph replay, an HMC trajectory and NUTS posteriors (GPU tier)."""
import ctypes
import os
import subprocess

import pytest
import torch

import pyro_b200 as pyro
import pyro_b200.distributions as dist
from conftest import EMULATE, device
from pyro_b200 import _build
from pyro_b200 import _native as N
from pyro_b200.infer import HMC, MCMC, NUTS
from pyro_b200.infer.mcmc import GlmPotential, TracePotential
from pyro_b200.infer.mcmc.compile import recognise
from test_glm_group_potential import _lin, _recognised
from test_glm_group_potential import test_group_kernel_sass as _check_group_kernel_sass
from test_glm_slope_potential import FORMS, SCALES, _chain_state, _chains, _check_against_oracle, \
    _check_layout, _check_slopes, _data, _oracle_potential, slope_model

DEV = device()
WIDE_KINDS = ["Bernoulli", "Poisson", "Normal"]     # Binomial keeps its 128-column limit


def _sorted(X, g, y):
    """The rows ordered by group (stable): the posterior does not depend on the order of the rows."""
    order = torch.argsort(g, stable=True)
    return X[order].contiguous(), g[order].contiguous(), y[order].contiguous()


def _wide_data(kind, n, D, G, slopes=(2,), seed=0, dev="cpu"):
    return _sorted(*_data(kind, n, D, G, dev=dev, seed=seed, slopes=slopes))


# ---- CPU tier: recognition and layout ----------------------------------------------------------------------------
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_recognises_wide_group_effect(kind, form, scale):
    """5 + 70 (1 + 1) = 145 columns with the rows sorted by group: GlmPotential, promised sorted."""
    G, slopes = 70, ((form, scale, 2),)
    X, g, y = _wide_data(kind, 400, 5, G)
    model = slope_model(kind, slopes, a_form="noncentred" if form == "centred" else "centred", G=G)
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), (kind, form, scale)
    assert pot.group_effect.G == G and pot.group_effect.sorted == 1
    _check_slopes(pot, slopes, G)
    assert torch.equal(pot.groups.cpu(), g.to(torch.int32))
    _check_layout(pot, model, (X, g, y))


SHAPES = {"radon": (919, 2, 85, ((("noncentred", "HalfCauchy", 1),))),
          "G1000": (3000, 3, 1000, ()),
          "S3": (600, 6, 50, (("centred", "const", 1), ("noncentred", "HalfNormal", 3), ("centred", "const", 5))),
          "D128": (500, 128, 4, ())}


@pytest.mark.parametrize("case", list(SHAPES))
def test_recognises_wide_shapes(case):
    n, D, G, slopes = SHAPES[case]
    X, g, y = _wide_data("Normal", n, D, G, slopes=[c for _, _, c in slopes])
    model = slope_model("Normal", slopes, a_scale="HalfNormal", G=G, sigma="latent")
    pot = _recognised(model, X, g, y)
    assert isinstance(pot, GlmPotential), case
    assert D + G * (1 + len(slopes)) > 128 and pot.group_effect.sorted == 1
    _check_slopes(pot, slopes, G)
    _check_layout(pot, model, (X, g, y))


def _softmax_group_model(X, g, y):
    """Softmax regression with a varying intercept by group (a wide, sorted index)."""
    D, K = X.shape[-1], 3
    W = pyro.sample("W", dist.Normal(X.new_zeros(K, D), 1.0).to_event(2))
    b = pyro.sample("b", dist.Normal(X.new_zeros(K), 10.0).to_event(1))
    a = pyro.sample("alpha", dist.Normal(X.new_zeros(70), 0.7).to_event(1))
    logits = X @ W.transpose(-1, -2) + b.unsqueeze(-2) + a[..., g].unsqueeze(-1)
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Categorical(logits=logits), obs=y)


def _latent_scale_group_model(X, g, y):
    """Logistic regression with a hierarchical weight scale tau and a varying intercept by group."""
    D = X.shape[-1]
    tau = pyro.sample("tau", dist.HalfNormal(X.new_full((), 1.0)))
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), tau.unsqueeze(-1)).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    a = _chains(pyro.sample("alpha", dist.Normal(X.new_zeros(70), 0.7).to_event(1)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_lin(X, w, b) + a[..., g]), obs=y)


@pytest.mark.parametrize("change", ["swapped_pair", "G65537", "D129", "mask", "fp64", "binomial", "softmax",
                                    "latent_weight_scale"])
def test_wide_near_misses_are_not_recognised(change):
    kind, n, D, G, slopes = "Bernoulli", 400, 5, 70, (("centred", "HalfNormal", 2),)
    if change in ("softmax", "latent_weight_scale"):   # 5 + 70 = 75 columns would fit: make it 200 + 70 wide
        X, g, y = _wide_data(kind, n, 60, G, slopes=())
        X = torch.cat([X, X, X, X[:, :20]], 1).contiguous()   # D = 200 > 128 - G
        if change == "softmax":
            y = torch.randint(0, 3, (n,), generator=torch.Generator().manual_seed(3))
            model = _softmax_group_model
        else:
            X = X[:, :100].contiguous()                       # D = 100: 100 + 70 = 170 columns
            model = _latent_scale_group_model
        assert not isinstance(_recognised(model, X, g, y), GlmPotential), change
        return
    if change == "binomial":
        kind = "Binomial"
    if change == "D129":
        D = 129
    if change == "G65537":
        G = 65537
    X, g, y = _wide_data(kind, n, D, G)
    if change == "swapped_pair":            # one descending pair: the index is not sorted
        i = int((g[1:] > g[:-1]).nonzero()[0])
        g = g.clone()
        g[i], g[i + 1] = g[i + 1].clone(), g[i].clone()
    if change == "fp64":
        X, y = X.double(), y.double()
    model = slope_model(kind, slopes, G=G, change="mask" if change == "mask" else None)
    assert not isinstance(_recognised(model, X, g, y), GlmPotential), change
    if change == "swapped_pair":            # sorted, the same model is recognised
        X, g, y = _wide_data(kind, n, D, G)
        assert isinstance(_recognised(model, X, g, y), GlmPotential)


def test_narrow_models_are_promised_sorted_only_when_they_are():
    """At <= 128 columns the flag is set from the data but not read: an unsorted index keeps the one-hot route."""
    X, g, y = _data("Poisson", 300, 5, 6)
    pot = _recognised(slope_model("Poisson", (), G=6), X, g, y)
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 0
    pot = _recognised(slope_model("Poisson", (), G=6), *_sorted(X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1


def test_wide_entry_point_validates_arguments_before_any_cuda_call():
    L = N.lib()
    p = ctypes.c_void_p(4096)

    def regression(D=10, G=40, S=2, srt=1, kind=N.GLM_POISSON, n=10000, groups=p, scale=False):
        # z = [w (D), b, alpha (G), beta_1 (G), .., beta_S (G)]
        e = N.b2_glm_group_effect()
        e.groups, e.G, e.a_off, e.noncentred, e.s_off, e.s_const = groups, G, D + 1, 0, -1, 0.7
        e.S, e.sorted = S, srt
        for k in range(min(S, 3)):
            s = e.slope[k]
            s.col, s.b_off, s.s_off, s.noncentred, s.s_const = k, D + 1 + (k + 1) * G, -1, 0, 0.5
        m = N.b2_glm_regression(kind=kind, X=p, y=p, N=n, D=D, K=1, trials=p, has_bias=1, w_off=0, b_off=D,
                                s_w=1.0, s_b=10.0, s_off=-1, sigma=1.0, group=ctypes.pointer(e))
        if scale:
            sc = N.b2_glm_weight_scale(tau_off=D + 1 + G * (1 + S), lam_off=-1, tau_prior=N.SIGMA_HALFNORMAL,
                                       tau_p0=1.0)
            m.scale = ctypes.pointer(sc)
            m._keep = sc
        m._keep_e = e
        return m, D + 1 + G * (1 + min(S, 3)) + (1 if scale else 0)

    def call(C=4, **kw):
        m, Dz = regression(**kw)
        return L.b2_glm_potential(ctypes.byref(m), p, C, Dz, p, p, None, 0, None)

    def workspace(C=4, **kw):
        return L.b2_glm_potential_workspace(ctypes.byref(regression(**kw)[0]), C)

    assert call() == -5                                   # 10 + 40 * 3 = 130 columns, sorted: the workspace is next
    assert call(srt=0) == -2                              # unsorted past 128 columns
    assert call(srt=0, G=39) == -5 and call(srt=1, G=39) == -5
    assert call(srt=2) == -2 and call(srt=-1) == -2 and call(srt=2, G=39) == -2
    assert call(S=0, G=65536) == -5 and call(S=0, G=65537) == -2
    assert call(D=129) == -2 and call(S=4) == -2 and call(kind=N.GLM_CATEGORICAL) == -2
    assert call(kind=N.GLM_NORMAL) == -5 and call(kind=N.GLM_BINOMIAL) == -2
    assert call(scale=True) == -2
    assert call(groups=ctypes.c_void_p(4100)) == -2
    # the workspace grows with G and C, not with N (past one CTA per SM)
    assert workspace() > 256 and workspace(srt=0) == 256
    assert workspace(G=80) > workspace(G=40) and workspace(C=200) > workspace(C=4)
    assert workspace(n=10_000_000) == workspace(n=20_000_000)


# ---- CPU tier: what ptxas makes of the gathered kernels ----------------------------------------------------------
FAMILIES = ["9BernoulliE", "7PoissonE", "6NormalE"]
GATHER_KERNELS = ["glm_group_gather_tc_kernelINS_2tc%sLi%dE" % (f, dc) for f in FAMILIES for dc in (1, 2, 3, 4)]


@pytest.fixture(scope="module")
def gather_sass(tmp_path_factory):
    import test_glm_tc_sass as sass_test
    nvcc, cuobjdump = sass_test._tools()
    obj = str(tmp_path_factory.mktemp("glm_gather_sass") / "glm_group_gather_tc.o")
    src = os.path.join(_build.CSRC, "glm_group_gather_tc.cu")
    r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return {"glm_group_gather_tc": (r.stdout + r.stderr, sass)}


@pytest.mark.parametrize("mangled", GATHER_KERNELS)
def test_gather_kernel_sass(gather_sass, mangled):
    """No C7515/C7520 serialisation note, no spills, no stack frame, and each GEMM one HGMMA chain with one wait."""
    import test_glm_tc_sass as sass_test
    _check_group_kernel_sass(gather_sass, "glm_group_gather_tc", mangled)
    props, _ = sass_test._ptxas_properties(gather_sass["glm_group_gather_tc"][0], mangled)
    assert "0 bytes stack frame" in props, props


# ---- GPU tier ------------------------------------------------------------------------------------------------------
def _gpu():
    if EMULATE:
        pytest.skip("kernel test")


@pytest.mark.gpu
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_potential_against_fp64_and_trace(kind, form, scale):
    """7 + 70 (1 + 1) = 147 columns: U and dU/dz for C = 1, 64, 65 against fp64 and TracePotential, bitwise
    repeatable."""
    _gpu()
    n, D, G = 9000, 7, 70
    X, g, y = _wide_data(kind, n, D, G, seed=n + D, dev=DEV)
    model = slope_model(kind, ((form, scale, 2),), a_scale="HalfNormal", G=G,
                        sigma="latent" if scale == "HalfCauchy" else "const")
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1, (kind, form, scale)
    _check_against_oracle(model, pot, X, g, y, kind, (1, 64, 65), 0, "wide %s %s %s" % (kind, form, scale))


RAGGED_N = [1, 63, 64, 65, 10_003, 250_001]
# partial last tiles that are the first, the second or a later tile of their warpgroup's range (D = 32: Q = 528)
PARTIAL_N = [10_003, 33_793, 67_600]
RAGGED_D = [2, 32, 33, 64, 65, 128]     # recognition needs D >= 2 with a group effect, whatever the width


@pytest.mark.gpu
@pytest.mark.parametrize("n", RAGGED_N)
@pytest.mark.parametrize("D", RAGGED_D)
def test_ragged_shapes(D, n):
    """Every atom count, tiles cut anywhere, S = 0 .. 3 and the kind cycling over the three; G = 150."""
    _gpu()
    i = RAGGED_D.index(D) + RAGGED_N.index(n)
    kind, form, S = WIDE_KINDS[i % 3], FORMS[(i // 3) % 2], min(i % 4, D)
    G = 150
    slopes = tuple((FORMS[(i + k) % 2], "HalfNormal" if k == 0 else "const", D - 1 - k) for k in range(S))
    X, g, y = _wide_data(kind, n, D, G, slopes=[c for _, _, c in slopes], seed=i, dev=DEV)
    model = slope_model(kind, slopes, a_form=form, a_scale="HalfNormal", G=G)
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == S, (kind, D, S, n)
    _check_against_oracle(model, pot, X, g, y, kind, (1, 65), 1, "%s D=%d S=%d n=%d" % (kind, D, S, n),
                          gtol=5e-4 if n >= 8192 else 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("n", PARTIAL_N)
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_partial_last_tile_anywhere_in_its_range(kind, n):
    """A partial last tile after other tiles of the same warpgroup's range: U and the bias gradient take every row
    once."""
    _gpu()
    X, g, y = _wide_data(kind, n, 32, 150, slopes=(), seed=6, dev=DEV)
    model = slope_model(kind, (), a_scale="HalfNormal", G=150)
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1
    _check_against_oracle(model, pot, X, g, y, kind, (1, 65), 4, "%s n=%d" % (kind, n))


def _layout(case):
    """(n, D, G, S, g): one group over many tiles and ranges; every group one row; mostly empty groups; runs that end
    on every tile boundary (and so on every range boundary)."""
    gen = torch.Generator().manual_seed(4)
    if case == "one_big_group":
        n, D, G, S = 250_001, 120, 5, 1
        g = torch.cat([torch.zeros(200_000, dtype=torch.int64), torch.randint(1, G, (n - 200_000,), generator=gen)])
    elif case == "single_rows":
        n, D, G, S = 10_003, 4, 10_003, 0
        g = torch.arange(n)
    elif case == "empty_groups":
        n, D, G, S = 3000, 4, 5000, 1
        g = torch.randint(0, 40, (n,), generator=gen) * 117
    else:
        n, D, G, S = 64 * 600, 16, 600, 1
        g = torch.arange(n) // 64
    return n, D, G, S, g.sort().values


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["one_big_group", "single_rows", "empty_groups", "tile_boundaries"])
def test_run_layouts(case):
    _gpu()
    n, D, G, S, g = _layout(case)
    kind = "Normal" if case in ("one_big_group", "tile_boundaries") else "Bernoulli"
    X, _, y = _data(kind, n, D, 2, seed=9, slopes=())
    slopes = (("noncentred", "HalfNormal", D - 1),) if S else ()
    X, g, y = X.to(DEV), g.to(DEV), y.to(DEV)
    model = slope_model(kind, slopes, a_scale="HalfNormal", G=G)
    pot = recognise(model, (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1, case
    _check_against_oracle(model, pot, X, g, y, kind, (1, 65), 2, case, gtol=5e-4 if n >= 8192 else 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_bad_index_and_descending_pair_give_nan(kind):
    """An index outside [0, G) makes U and the group gradients NaN; a descending pair makes U NaN for every chain; the
    next valid call is exact again."""
    _gpu()
    slopes = (("centred", "HalfCauchy", 1), ("noncentred", "const", 4))
    X, g, y = _wide_data(kind, 20_000, 6, 60, slopes=(1, 4), seed=5, dev=DEV)
    pot = recognise(slope_model(kind, slopes, a_scale="HalfCauchy", G=60), (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1
    z = _chain_state(pot, 8, 0)
    U0, G0 = pot.value_and_grad(z)
    for bad in (60, -1, 1 << 30):
        pot.groups[4321] = bad
        U, G = pot.value_and_grad(z)
        torch.cuda.synchronize()
        assert bool(torch.isnan(U).all()), bad
        for site in ("alpha", "beta_b1", "eta_b2"):
            assert bool(torch.isnan(G[:, pot.sites[site][0]]).all()), (bad, site)
        pot.groups[4321] = int(g[4321])
    for i in (4321, 64 * 37 - 1, 0):          # inside a tile, across a tile boundary, the first row
        a, b = int(pot.groups[i]), int(pot.groups[i + 1])
        pot.groups[i], pot.groups[i + 1] = b + 1, a
        U, _ = pot.value_and_grad(z)
        torch.cuda.synchronize()
        assert bool(torch.isnan(U).all()), i
        pot.groups[i], pot.groups[i + 1] = a, b
    U1, G1 = pot.value_and_grad(z)
    assert torch.equal(U1, U0) and torch.equal(G1, G0)


@pytest.mark.gpu
def test_unsorted_wide_index_raises():
    _gpu()
    X, g, y = _data("Poisson", 3000, 5, 200, dev=DEV)          # 5 + 200 columns
    sites = {"w": (slice(0, 5), "identity", (5,)), "b": (slice(5, 6), "identity", ()),
             "alpha": (slice(6, 206), "identity", (200,))}
    group = {"site": "alpha", "index": g, "noncentred": False, "s_const": 0.7}
    with pytest.raises(ValueError):
        GlmPotential(X, y, "Poisson", sites, "w", "b", group=group)
    Xs, gs, ys = _sorted(X, g, y)
    pot = GlmPotential(Xs, ys, "Poisson", sites, "w", "b", group=dict(group, index=gs))
    assert pot.group_effect.sorted == 1


@pytest.mark.gpu
def test_sorted_flag_does_not_move_the_one_hot_route():
    """At <= 128 columns U and dU/dz are bitwise the same with the flag 0 and 1."""
    _gpu()
    slopes = (("noncentred", "HalfNormal", 3),)
    X, g, y = _wide_data("Bernoulli", 30_000, 8, 40, slopes=(3,), seed=3, dev=DEV)
    pot = recognise(slope_model("Bernoulli", slopes, a_scale="HalfNormal", G=40), (X, g, y))
    assert pot.group_effect.sorted == 1 and 8 + 40 * 2 <= 128
    z = _chain_state(pot, 65, 0)
    U1, G1 = pot.value_and_grad(z)
    pot.group_effect.sorted = 0
    U0, G0 = pot.value_and_grad(z)
    assert torch.equal(U0, U1) and torch.equal(G0, G1)


@pytest.mark.gpu
def test_captured_graph_replay_equals_eager():
    _gpu()
    slopes = (("noncentred", "HalfNormal", 3), ("centred", "const", 9))
    X, g, y = _wide_data("Normal", 70001, 16, 200, slopes=(3, 9), seed=3, dev=DEV)
    pot = recognise(slope_model("Normal", slopes, a_scale="HalfNormal", G=200, sigma="latent"), (X, g, y))
    assert pot.group_effect.S == 2 and pot.group_effect.sorted == 1
    z = _chain_state(pot, 64, 0)
    U0, G0 = pot.value_and_grad(z)
    zbuf = torch.zeros_like(z)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pot.value_and_grad(zbuf)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    n0 = N.launch_count()
    with torch.cuda.graph(graph):
        Ug, Gg = pot.value_and_grad(zbuf)
    assert N.launch_count() - n0 == 4   # pack, GLM kernel, GLM finish, potential finish
    zbuf.copy_(z)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(Ug, U0) and torch.equal(Gg, G0)


@pytest.mark.gpu
def test_hmc_trajectory_matches_oracle_integrator():
    _gpu()
    from oracle import mcmc as omcmc
    n, C, L, eps = 8192, 4, 20, 0.004
    slopes = (("noncentred", "HalfCauchy", 2), ("centred", "const", 5))
    X, g, y = _wide_data("Bernoulli", n, 8, 60, slopes=(2, 5), seed=11, dev=DEV)
    pot = recognise(slope_model("Bernoulli", slopes, a_scale="HalfNormal", G=60), (X, g, y))
    assert isinstance(pot, GlmPotential) and pot.group_effect.sorted == 1
    kernel = HMC(potential_fn=pot, step_size=eps, num_steps=L, adapt_step_size=False)
    z0 = _chain_state(pot, C, 5)
    r0 = torch.randn(C, pot.dim, device=DEV)
    z, r = z0.clone(), r0.clone()
    _, gr = pot.value_and_grad(z)
    epsv = torch.full((C,), eps, device=DEV)
    minv = torch.ones(C, pot.dim, device=DEV)
    for _ in range(L):
        z, r, gr, U, _ = kernel._leapfrog(z, r, gr, epsv, minv)
    Uo = _oracle_potential(X.cpu(), g.cpu(), y.cpu(), pot, "Bernoulli")
    for c in range(C):
        zr, rr, _, ur = omcmc.velocity_verlet(z0[c].double().cpu(), r0[c].double().cpu(), Uo,
                                              torch.ones(pot.dim, dtype=torch.float64), eps, num_steps=L)
        ez = float((z[c].double().cpu() - zr).abs().max())
        er = float((r[c].double().cpu() - rr).abs().max()) / max(1.0, float(rr.abs().max()))
        eu = abs(float(U[c]) - float(ur)) / max(1.0, abs(float(ur)))
        assert ez <= 1e-4 and er <= 5e-4 and eu <= 2e-5, (ez, er, eu)


def radon85(X, g, y):
    """Varying intercept and a varying slope on the floor column (1) over 85 counties, non-centred, latent sigma."""
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    sigma = pyro.sample("sigma", dist.HalfNormal(X.new_full((), 1.5)))
    s_a = pyro.sample("s_a", dist.HalfCauchy(X.new_full((), 1.0)))
    eta_a = pyro.sample("eta_a", dist.Normal(X.new_zeros(85), 1.0).to_event(1))
    s_b = pyro.sample("s_b", dist.HalfCauchy(X.new_full((), 0.5)))
    eta_b = pyro.sample("eta_b", dist.Normal(X.new_zeros(85), 1.0).to_event(1))
    a = _chains(s_a.unsqueeze(-1) * eta_a)
    beta = _chains(s_b.unsqueeze(-1) * eta_b)
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Normal(_lin(X, w, b) + a[..., g] + beta[..., g] * X[:, 1], sigma), obs=y)


def multilevel_logistic500(X, g, y):
    D = X.shape[-1]
    w = pyro.sample("w", dist.Normal(X.new_zeros(D), 1.0).to_event(1))
    b = pyro.sample("b", dist.Normal(X.new_zeros(()), 10.0))
    s_a = pyro.sample("s_a", dist.HalfNormal(X.new_full((), 1.0)))
    alpha = _chains(pyro.sample("alpha", dist.Normal(X.new_zeros(500), s_a.unsqueeze(-1)).to_event(1)))
    s_1 = pyro.sample("s_1", dist.HalfNormal(X.new_full((), 0.5)))
    beta_1 = _chains(pyro.sample("beta_1", dist.Normal(X.new_zeros(500), s_1.unsqueeze(-1)).to_event(1)))
    with pyro.plate("data", X.shape[0]):
        pyro.sample("y", dist.Bernoulli(logits=_lin(X, w, b) + alpha[..., g] + beta_1[..., g] * X[:, 0]), obs=y)


def _radon_data(seed):
    """919 rows over 85 counties of uneven size (a few large, many small), sorted by county; D = 2 with the floor
    column 0 or 1."""
    gen = torch.Generator().manual_seed(seed)
    sizes = torch.distributions.Categorical(probs=torch.rand(85, generator=gen) ** 3 + 0.01)
    torch.manual_seed(seed)
    g = sizes.sample((919,)).sort().values
    X, _, y = _data("Normal", 919, 2, 2, seed=seed, slopes=())
    X[:, 1] = (X[:, 1] > 0.5).to(X.dtype)
    a = 0.5 * torch.randn(85, generator=gen)
    bt = 0.3 * torch.randn(85, generator=gen)
    y = X @ torch.tensor([0.4, -0.6]) + 1.0 + a[g] + bt[g] * X[:, 1] + 0.6 * torch.randn(919, generator=gen)
    return X.to(DEV), g.to(DEV), y.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["radon85", "multilevel_logistic500"])
def test_nuts_posterior_matches_trace_potential(case):
    """NUTS with 8 chains on GlmPotential against TracePotential: means within 0.3 sd, sds within 25 %."""
    _gpu()
    if case == "radon85":
        model, (X, g, y) = radon85, _radon_data(22)
    else:
        model = multilevel_logistic500
        X, g, y = _wide_data("Bernoulli", 20_000, 6, 500, slopes=(0,), seed=21, dev=DEV)
    out = {}
    for compile_model in (True, False):
        kernel = NUTS(model, max_tree_depth=5)
        kernel.compile_model = compile_model
        # radon's county scales mix slowly: twice the draws keep the comparison's own noise inside the tolerances
        draws = 400 if case == "radon85" else 200
        mc = MCMC(kernel, num_samples=draws, warmup_steps=150, num_chains=8, seed=1 if compile_model else 2)
        mc.run(X, g, y)
        want = GlmPotential if compile_model else TracePotential
        assert type(kernel.potential) is want, type(kernel.potential).__name__
        if compile_model:
            assert kernel.potential.group_effect.S == 1 and kernel.potential.group_effect.sorted == 1
        s = mc.get_samples()
        cols = [s[name].reshape(s[name].shape[0], -1).double().cpu() for name in sorted(s)]
        out[compile_model] = torch.cat([c.log() if name.startswith("s_") or name == "sigma" else c
                                        for name, c in zip(sorted(s), cols)], -1)
    got, ref = out[True], out[False]
    m_, sd = got.mean(0), got.std(0)
    rm, rs = ref.mean(0), ref.std(0)
    print("\nnuts %s: max |mean diff| / sd %.2f, max |sd diff| / sd %.2f"
          % (case, float(((m_ - rm).abs() / rs).max()), float(((sd - rs).abs() / rs).max())))
    assert bool(((m_ - rm).abs() <= 0.3 * rs).all()), float(((m_ - rm).abs() / rs).max())
    assert bool(((sd - rs).abs() <= 0.25 * rs).all()), float(((sd - rs).abs() / rs).max())


@pytest.mark.gpu
def test_bind_nuts_recognises_reference_pyro_plate_radon():
    _gpu()
    from pyro_b200 import bind
    if not bind.add_reference_to_path():
        pytest.skip("reference Pyro is not built (oracle/_ref missing)")
    import pyro as ref_pyro
    import pyro.distributions as rdist
    from pyro.infer import MCMC as RefMCMC

    def radon(X, g, y):
        D = X.shape[-1]
        w = ref_pyro.sample("w", rdist.Normal(X.new_zeros(D), 1.0).to_event(1))
        b = ref_pyro.sample("b", rdist.Normal(X.new_zeros(()), 10.0))
        sigma = ref_pyro.sample("sigma", rdist.HalfNormal(X.new_full((), 1.5)))
        s_a = ref_pyro.sample("s_a", rdist.HalfCauchy(X.new_full((), 1.0)))
        s_b = ref_pyro.sample("s_b", rdist.HalfCauchy(X.new_full((), 0.5)))
        with ref_pyro.plate("county", 85):
            eta_a = ref_pyro.sample("eta_a", rdist.Normal(X.new_zeros(()), 1.0))
            beta = ref_pyro.sample("beta", rdist.Normal(X.new_zeros(()), s_b))
        with ref_pyro.plate("data", X.shape[0]):
            ref_pyro.sample("y", rdist.Normal(X @ w + b + s_a * eta_a[g] + beta[g] * X[:, 1], sigma), obs=y)

    args = _radon_data(2)
    pot = bind.recognise(radon, args, {}, poutine=ref_pyro.poutine)
    assert isinstance(pot, GlmPotential) and pot.group_effect.S == 1 and pot.group_effect.sorted == 1
    kernel = bind.NUTS(radon, num_chains=4, seed=0)
    mc = RefMCMC(kernel, num_samples=20, warmup_steps=20, num_chains=1, disable_progbar=True)
    mc.run(*args)
    assert isinstance(kernel._kernel.potential, GlmPotential)
