"""``mu.prot`` -- CITE-seq protein modality (reference muon/prot.py, muon/_prot/__init__.py)."""
from . import pp  # noqa: F401
