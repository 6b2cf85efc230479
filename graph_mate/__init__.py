"""`graph_mate` import shim: the reference's Python module name (crates/mate, graph_mate.pyi) bound to
the H100 implementation, so `from graph_mate import DiGraph, Graph, Layout, FileFormat` — the imports of
crates/mate/tests/*.py and of the reference's notebooks — resolve to graph_b200 unchanged."""
from graph_b200 import (DiGraph, FileFormat, Graph, Layout, PageRankResult,  # noqa: F401
                        TriangleCountResult, WccResult)

__all__ = ["DiGraph", "Graph", "Layout", "FileFormat", "PageRankResult", "WccResult", "TriangleCountResult"]
