"""TEST INFRASTRUCTURE ONLY: CPU restatement of the reference's hot path (the parity checker).

Nothing under ``oracle/`` is imported by the product package ``videosys_b200``.  Allowed importers:
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs.
Parity pinning: the reference's own tests hold no golden vectors for this path (SURVEY.md section 4);
the oracle is pinned by (1) executing the unmodified reference modules in the authoring container
(tests/test_oracle_vs_reference.py, skipped where the reference tree is absent) and (2) golden vectors
generated from the reference by oracle/gen_golden.py and committed under tests/golden/.
"""
