"""CPU oracle for the two hot paths (EnCodec SEANet+RVQ, MusicGen LM decode).

TEST INFRASTRUCTURE ONLY -- never imported by the product package `audiocraft_b200`.
Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs may import it, and only as the checker / the timed CPU baseline.

Each function is a plain fp32 PyTorch-on-CPU restatement of the reference algorithm and cites
the reference file:line it follows (paths relative to the reference source tree).  The restatement is
pinned against the real reference modules run on the CPU (oracle/ref_import.py,
tests/golden/make_golden.py -> tests/golden/*.pt; tests/test_oracle_vs_golden.py), because the
reference's own tests hold no numeric golden vectors for this path (SURVEY.md section 4 / 8c).
"""
