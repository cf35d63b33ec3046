"""grakel_b200 -- H100-native graph-kernel Gram engine behind the GraKeL operator API.

Hot path only: WeisfeilerLehman (subtree, or over EdgeHistogram / ShortestPath), VertexHistogram,
EdgeHistogram, ShortestPath, ShortestPathAttr, WeisfeilerLehmanOptimalAssignment, GraphHopper, NeighborhoodHash, RandomWalk,
RandomWalkLabeled, Propagation, PropagationAttr, PyramidMatch, HadamardCode, NeighborhoodSubgraphPairwiseDistance, SubgraphMatching,
OddSth, MultiscaleLaplacian, SvmTheta, GraphletSampling, CoreFramework
(`fit` / `transform` / `fit_transform` / `diagonal`), plus the `GraphKernel` name dispatcher.  All kernel matrices are computed by
hand-written sm_90a CUDA (`libgrakel_b200.so`, C-ABI in include/grakel_b200.h); there is no CPU path.
"""
from .packing import Graph
from .kernels import (EdgeHistogram, GraphHopper, GraphletSampling, HadamardCode, Kernel, MultiscaleLaplacian, NeighborhoodHash,
                      NeighborhoodSubgraphPairwiseDistance, OddSth, Propagation, PropagationAttr, PyramidMatch,
                      RandomWalk, SubgraphMatching, SvmTheta, _dirac,
                      RandomWalkLabeled, ShortestPath, ShortestPathAttr, VertexHistogram, WeisfeilerLehman,
                      WeisfeilerLehmanOptimalAssignment)
from .core_framework import CoreFramework
from .graph_kernels import GraphKernel
from ._lib import default_device, set_default_device

__version__ = "0.1.0"
__all__ = ["Graph", "Kernel", "GraphKernel", "WeisfeilerLehman", "VertexHistogram", "ShortestPath",
           "ShortestPathAttr", "EdgeHistogram", "CoreFramework", "WeisfeilerLehmanOptimalAssignment", "GraphHopper",
           "NeighborhoodHash", "RandomWalk", "RandomWalkLabeled", "Propagation", "PropagationAttr", "PyramidMatch",
           "HadamardCode", "NeighborhoodSubgraphPairwiseDistance", "SubgraphMatching", "OddSth", "MultiscaleLaplacian",
           "SvmTheta", "GraphletSampling", "set_default_device",
           "default_device"]
