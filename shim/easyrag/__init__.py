"""Overlay of the reference's ``easyrag`` package: put this directory's parent (``<repo>/shim``) on ``sys.path``
BEFORE the reference's ``src`` and ``pipeline/pipeline.py`` runs unchanged against the H100 classes.

``pipeline.py:15,19`` import ``..custom.embeddings`` and ``..custom.retrievers`` relative to the ``easyrag``
package.  This package extends its search path with every other ``easyrag`` directory on ``sys.path`` (the
reference's), so ``easyrag.pipeline.*``, ``easyrag.utils.*`` and the rest of ``easyrag.custom.*`` still come from
the reference while the two modules below resolve here first.
"""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
