"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the reference algorithms on the two hot paths of pyro-ppl/pyro 1.9.1
(Trace_ELBO SVI step; NUTS/HMC leapfrog), each function citing the reference file:line it follows.
Parity is PINNED: tests/test_oracle_golden.py checks every function here against golden vectors
produced by the UNMODIFIED reference (tests/golden/make_golden.py) and against the reference's own
test fixtures.

Only tests/, __graft_entry__ (smoke(), and build() for oracle/build_ref.py) and bench.py's
CPU-baseline legs may import this package;
pyro_b200/ never does (tests/test_layout.py enforces it).
"""
