"""CPU oracle for the DDPM noise-prediction hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is product code: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it, and only as the checker / CPU baseline.

PARITY UNPINNED: the reference (magenta/symbolic-music-diffusion) ships no tests
or golden vectors and its JAX 0.2.8 / flax 0.3.0 stack cannot be installed here,
so the restatement is pinned only by (a) the published JAX threefry / PRNG
known-answer values, (b) analytic known-answer cases, and (c) fp32-vs-fp64
self-consistency.
"""
