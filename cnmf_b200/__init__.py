"""cnmf_b200 -- GPU-native consensus NMF: the factorize -> combine -> consensus hot path of dylkot/cNMF
on hand-written sm_90a (H100) CUDA behind the reference's own class / CLI / file layout.

Exports mirror the reference package (`src/cnmf/__init__.py:1-2`).
Importing this package needs neither a GPU nor the compiled library; using it does.
"""
from .io import load_df_from_npz, save_df_to_npz, save_df_to_text  # noqa: F401
from .pipeline import cNMF, main  # noqa: F401
from .preprocess import Preprocess  # noqa: F401

__version__ = "0.1.0"
