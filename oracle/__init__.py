"""oracle/ -- TEST INFRASTRUCTURE, not product code.

CPU restatement of the reference hot path (dylkot/cNMF `factorize -> combine ->
consensus`, whose arithmetic lives in the third-party scikit-learn 1.9.0 that the
image ships) used ONLY as the checker:

  * ``tests/``                      -- parity tests compare the CUDA path against it
  * ``__graft_entry__.smoke()``     -- one tiny parity check on cuda:0
  * ``bench.py`` ``cpu_baseline``   -- and ``--impl reference`` time it on the host cores

Nothing under ``cnmf_b200/`` imports this package; the product path fails loudly
when its CUDA library is missing instead of falling back here.

Pinning status ("is the oracle trustworthy?"):
  * The reference's own tests hold NO offline golden vectors for this path
    (``tests/test_reproducibility.py:85-89`` bypasses factorize; the consensus goldens
    are network downloads, ``download_pytest_data.py:38-52``; SURVEY.md section 8c).
  * Therefore the oracle is pinned against OUTPUTS OF THE REFERENCE ITSELF:
    ``oracle/make_golden.py`` imports ``src/cnmf/cnmf.py`` of a cNMF checkout (CNMF_REFERENCE)
    unmodified (through ``oracle/refshim.py``, a scanpy/matplotlib stub) and writes
    ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks every restatement in
    this package against those fixtures.

Modules
  refshim.py        loader for the unmodified reference module (needs CNMF_REFERENCE)
  make_golden.py    script that generated tests/golden/ (committed with the fixtures)
  nmf_ref.py        numpy restatement of sklearn's MU / CD NMF solvers + random init
  consensus_ref.py  numpy restatement of cNMF.consensus numerics
  reference_path.py the reference's factorize/consensus call sequence on sklearn
                    (runs anywhere scikit-learn is installed)
"""
