"""Golden fixtures of the Binomial family (same recipe as make_golden.py: the UNMODIFIED reference imported from
/root/reference + the opt_einsum stand-in; run in the build container):

    python tests/golden/make_golden_binomial.py

  binomial.npz  pyro.distributions.Binomial(total_count, logits | probs).log_prob (pyro/distributions/torch.py:83-101,
                log_binomial at tol = 0) and its autograd gradients with respect to the value, the logits or probs
                and total_count, in fp64 and fp32:
                  kat_*     the reference's Binomial fixtures (tests/distributions/conftest.py:810-831)
                  rand_*    random batches, n in 0..200, k in 0..n, logits ~ 3 N(0, 1)
                  edge_*    n = 0, k in {0, n}, |logits| up to 80, probs near 0 and 1
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "opt_einsum_standin"))
sys.path.insert(0, "/root/reference")

import pyro  # noqa: E402
import pyro.distributions as dist  # noqa: E402

assert pyro.__version__ == "1.9.1"


def score(n, k, param, kind, dtype):
    n = torch.as_tensor(n, dtype=dtype).clone().requires_grad_(True)
    k = torch.as_tensor(k, dtype=dtype).clone().requires_grad_(True)
    p = torch.as_tensor(param, dtype=dtype).clone().requires_grad_(True)
    d = dist.Binomial(n, **{kind: p}, validate_args=False)
    assert d.approx_log_prob_tol == 0.0
    lp = d.log_prob(k)
    gn, gp, gk = torch.autograd.grad(lp.sum(), [n, p, k])
    n, k, p = torch.broadcast_tensors(n, k, p)
    return {"n": n.detach().numpy(), "k": k.detach().numpy(), "p": p.detach().numpy(), "lp": lp.detach().numpy(),
            "dn": gn.expand(n.shape).numpy(), "dp": gp.expand(n.shape).numpy(), "dk": gk.expand(n.shape).numpy()}


def main():
    out = {}

    def put(name, n, k, param, kind):
        for dt, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
            for key, v in score(n, k, param, kind, dt).items():
                out["%s_%s_%s_%s" % (name, kind, tag, key)] = v.reshape(-1)

    # the reference fixtures (probs), and the same points through logits
    kat = [(8.0, [4.0], [0.6]), (8.0, [[2.0], [4.0]], [0.3]), (8.0, [[4.0], [3.0]], [[0.2], [0.4]]),
           ([0.0, 0.0], [[0.0, 0.0], [0.0, 0.0]], [0.2, 0.4]),
           ([[8.0, 7.0], [5.0, 9.0]], [[6.0, 3.0], [2.0, 8.0]], [0.2, 0.4])]
    ns, ks, ps = [], [], []
    for n, k, p in kat:
        n, k, p = torch.broadcast_tensors(torch.tensor(n, dtype=torch.float64), torch.tensor(k, dtype=torch.float64),
                                          torch.tensor(p, dtype=torch.float64))
        ns.append(n.reshape(-1)), ks.append(k.reshape(-1)), ps.append(p.reshape(-1))
    n, k, p = torch.cat(ns), torch.cat(ks), torch.cat(ps)
    put("kat", n, k, p, "probs")
    put("kat", n, k, torch.log(p) - torch.log1p(-p), "logits")

    g = torch.Generator().manual_seed(20261016)
    n = torch.randint(0, 201, (1000,), generator=g).double()
    k = torch.floor(torch.rand(1000, generator=g, dtype=torch.float64) * (n + 1)).clamp(max=n)
    l = 3 * torch.randn(1000, generator=g, dtype=torch.float64)
    put("rand", n, k, l, "logits")
    put("rand", n, k, torch.sigmoid(l).clamp(1e-6, 1 - 1e-6), "probs")

    n = torch.tensor([0, 0, 1, 1, 10, 10, 10, 10, 100, 100, 200, 200, 50, 50, 7, 7], dtype=torch.float64)
    k = torch.tensor([0, 0, 0, 1, 0, 10, 10, 0, 100, 0, 200, 0, 25, 25, 3, 4], dtype=torch.float64)
    l = torch.tensor([0.0, -80.0, 80.0, -80.0, -80.0, 80.0, -40.0, 40.0, 80.0, -80.0, 30.0, -30.0, 0.0, 1e-3,
                      -5.0, 5.0], dtype=torch.float64)
    put("edge", n, k, l, "logits")
    pr = torch.tensor([0.5, 1e-12, 1 - 1e-12, 1e-9, 1e-6, 1 - 1e-6, 0.999, 0.001, 1 - 1e-4, 1e-4, 0.9, 0.1, 0.5,
                       0.5, 0.3, 0.7], dtype=torch.float64)
    put("edge", n, k, pr, "probs")
    np.savez_compressed(os.path.join(HERE, "binomial.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
