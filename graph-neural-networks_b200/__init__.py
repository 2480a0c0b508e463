"""b200gf — H100-native LSIGF graph-filter path (drop-in for alegnn.utils.graphML.LSIGF / GraphFilter).

The directory is called `graph-neural-networks_b200` (not a valid Python identifier); import it through the
`gnn_b200` loader module at the repo root:  `import gnn_b200 as b200`.
"""
from . import _cabi  # noqa: F401
from .gso import SparseGSO, Plan, plan_for, clear_plan_cache  # noqa: F401
from .graphML import LSIGF, GraphFilter, install, uninstall, fuse_layers, to_node_major, to_feature_major, node_major_ld, padded_ld  # noqa: F401

from .edgevariant import EVGF, EdgeVariantGF, SparseEdgeVariantGF  # noqa: F401,E402
from .pooling import MaxPoolLocal  # noqa: F401,E402
from .activations import MaxLocalActivation, MedianLocalActivation, NoActivation  # noqa: F401,E402
from .recurrent import GatedGRNN, HiddenState, TimeGatedHiddenState, NodeGatedHiddenState  # noqa: F401,E402
from .edgegated import EdgeGatedGRNN, EdgeGatedHiddenState, EdgeGatePattern  # noqa: F401,E402
from .nodevariant import NVGF, NodeVariantGF, TapMap, copy_nodes  # noqa: F401,E402
from .arma import jARMA, GraphFilterARMA, ArmaOperator  # noqa: F401,E402
from .attention import (graphAttention, graphAttentionLSIGF, graphAttentionEVGF, GraphAttentional,  # noqa: F401,E402
                        GraphFilterAttentional, EdgeVariantAttentional)
from .delayed import LSIGF_DB, GraphFilter_DB, GRNN_DB, HiddenState_DB  # noqa: F401,E402
from .aggregation import AggregationGNN, MultiNodeAggregationGNN, AggregationOperator  # noqa: F401,E402
from .graphed import graphed, GraphedForward  # noqa: F401,E402

__all__ = ["EVGF", "EdgeVariantGF", "MaxPoolLocal", "LSIGF", "GraphFilter", "SparseGSO", "Plan", "plan_for", "install", "uninstall", "fuse_layers"]
