"""``easyrag.custom`` overlay: ``retrievers``, ``embeddings`` and ``compressors`` come from easyrag_b200, every other
module (rerankers, hierarchical, template, ...) from the reference's own ``easyrag/custom`` directory."""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
