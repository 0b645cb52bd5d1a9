"""harmony_b200 — H100-native (sm_90a) implementation of the Harmony hot loop.

Host side mirrors the reference's R surface (RunHarmony / harmonize / the ``harmony`` module
class); all arithmetic on cell matrices runs in hand-written CUDA behind include/harmony_b200.h.
Importing this package does not load the CUDA library; constructing ``harmony`` does, and fails
loudly if it is missing (there is no CPU fallback).
"""
from .clustering import kmeans, nmi_ari, nmi_ari_cluster_labels_kmeans  # noqa: F401
from .community import leiden, nmi_ari_cluster_labels_leiden, umap_connectivities  # noqa: F401
from .graph import graph_components, graph_connectivity  # noqa: F401
from .harmony_option import harmony_options  # noqa: F401
from .kbet import kbet  # noqa: F401
from .lisi import compute_lisi  # noqa: F401
from .mapping import HarmonyReference  # noqa: F401
from .neighbors import TransferLabels, knn  # noqa: F401
from .pcr import pcr, pcr_comparison  # noqa: F401
from .silhouette import silhouette_batch, silhouette_label, silhouette_samples  # noqa: F401
from .ui import MapQuery, RunHarmony, prepare_inputs  # noqa: F401
from .utils import HarmonyConvergencePlot, harmonize  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    if name == "harmony":
        from .harmony import harmony
        return harmony
    raise AttributeError(name)
