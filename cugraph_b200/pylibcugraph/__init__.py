"""Python surface mirroring `pylibcugraph` for the PageRank / BFS / SSSP path
(reference python/pylibcugraph/pylibcugraph/__init__.py).  Same names, argument order and error
behaviour; device arrays go in as anything exposing `__cuda_array_interface__` (torch CUDA tensors,
cupy, numba) and come back as torch CUDA tensors (cupy is not a dependency here)."""
from cugraph_b200.pylibcugraph.exceptions import FailedToConvergeError
from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
from cugraph_b200.pylibcugraph.graph_properties import GraphProperties
from cugraph_b200.pylibcugraph.graphs import SGGraph
from cugraph_b200.pylibcugraph.algorithms import (pagerank, personalized_pagerank, bfs, sssp, katz_centrality, eigenvector_centrality, hits,
                                                  betweenness_centrality, edge_betweenness_centrality, select_random_vertices,
                                                  weakly_connected_components, strongly_connected_components,
                                                  generate_rmat_edgelist, in_degrees, out_degrees, degrees)

from cugraph_b200.pylibcugraph import utilities  # noqa: F401

__version__ = "26.10.00+b200"   # the reference version this surface mirrors (rapidsai/cugraph 26.10) + the build tag
__git_commit__ = ""             # only non-empty in a built distribution, as in the reference

__all__ = ["FailedToConvergeError", "ResourceHandle", "GraphProperties", "SGGraph",
           "pagerank", "personalized_pagerank", "bfs", "sssp", "katz_centrality", "eigenvector_centrality", "hits", "betweenness_centrality", "edge_betweenness_centrality", "select_random_vertices", "weakly_connected_components", "strongly_connected_components", "generate_rmat_edgelist", "in_degrees", "out_degrees", "degrees"]
