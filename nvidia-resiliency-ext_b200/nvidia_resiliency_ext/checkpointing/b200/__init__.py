"""The H100 snapshot engine: C-ABI binding (``_cabi``) and the host-side pipeline (``engine``)."""

from ._cabi import SnapError, library_path  # noqa: F401
