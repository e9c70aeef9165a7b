"""oracle/ — TEST INFRASTRUCTURE ONLY.

CPU restatement (numpy / torch-CPU) of the reference algorithm on the hot path, each function citing the
reference file:line it follows (paths relative to the reference repository's root).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this package; the product (3dgs-to-pc_b200/) never
does and has no CPU fallback.

Pinning: the reference ships no tests / golden vectors (SURVEY.md §4), so the oracle is pinned against outputs
of the UNMODIFIED reference run on a CPU through oracle/ref_shim.py; those outputs are committed
under tests/golden/ together with the generating script (tests/golden/make_golden.py).
"""
