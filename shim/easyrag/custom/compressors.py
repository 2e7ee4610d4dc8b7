"""Drop-in for the reference's ``easyrag/custom/compressors.py`` (imported at pipeline.py:22)."""
from easyrag_b200.compress import ContextCompressor                              # noqa: F401
