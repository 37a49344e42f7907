"""pointmvsnet_b200 -- sm_90a implementation of PointMVSNet's PointFlow hot path.

Mirrors the reference's import surface (pointmvsnet/model.py:8-12):
    pointmvsnet_b200.networks            EdgeConv, EdgeConvNoC
    pointmvsnet_b200.functions.functions get_pixel_grids
    pointmvsnet_b200.functions.gather_knn gather_knn  (dgcnn_ext shim)
    pointmvsnet_b200.utils.feature_fetcher FeatureFetcher
    pointmvsnet_b200.utils.torch_utils   get_knn_3d
    pointmvsnet_b200.nn.mlp / nn.conv    SharedMLP, Conv1d
    pointmvsnet_b200.utils.io / utils.eval_file_logger   PFM / camera files, per-view outputs (test.py:76)
plus the new ``PointFlow`` module that replaces the ``point_flow`` closure
(pointmvsnet/model.py:150-295).  ``install_as_pointmvsnet()`` aliases these modules
under the reference's own names so an unchanged ``pointmvsnet/model.py`` imports them.
"""
__version__ = "0.1.0"


def install_as_pointmvsnet(reference_root=None):
    """Make ``import pointmvsnet.<hot-path module>`` resolve to this package.

    With ``reference_root`` (a checkout of callmeray/PointMVSNet) the rest of the
    reference package (model.py, dataset, config ...) is imported from there and only
    the hot-path modules are replaced, so the unchanged ``pointmvsnet/model.py`` runs on
    the sm_90a kernels.  Without it, stub parent packages are created and every module
    this package mirrors is aliased (enough for ``from pointmvsnet.utils.torch_utils
    import get_knn_3d`` style imports).  See INTEGRATION.md."""
    import importlib
    import sys
    import types
    hot = {
        "pointmvsnet.functions.dgcnn_ext": "pointmvsnet_b200.functions.dgcnn_ext",
        "pointmvsnet.functions.gather_knn": "pointmvsnet_b200.functions.gather_knn",
        "pointmvsnet.utils.feature_fetcher": "pointmvsnet_b200.utils.feature_fetcher",
        "pointmvsnet.utils.torch_utils": "pointmvsnet_b200.utils.torch_utils",
        # output side (the reference's versions use np.int / ndarray.tostring, gone from numpy 2)
        "pointmvsnet.utils.io": "pointmvsnet_b200.utils.io",
        "pointmvsnet.utils.eval_file_logger": "pointmvsnet_b200.utils.eval_file_logger",
    }
    extra = {
        "pointmvsnet.functions.functions": "pointmvsnet_b200.functions.functions",
        "pointmvsnet.networks": "pointmvsnet_b200.networks",
        "pointmvsnet.nn.conv": "pointmvsnet_b200.nn.conv",
        "pointmvsnet.nn.mlp": "pointmvsnet_b200.nn.mlp",
        "pointmvsnet.nn.init": "pointmvsnet_b200.nn.init",
    }
    if reference_root is not None:
        if reference_root not in sys.path:
            sys.path.insert(0, reference_root)
        import pointmvsnet.functions as pf  # the reference package itself
        import pointmvsnet.utils  # noqa: F401
        for ref_name, ours in hot.items():
            sys.modules[ref_name] = importlib.import_module(ours)
            parent, _, leaf = ref_name.rpartition(".")
            setattr(sys.modules[parent], leaf, sys.modules[ref_name])
        pf.dgcnn_ext = sys.modules["pointmvsnet.functions.dgcnn_ext"]
        import pointmvsnet.networks as ref_networks
        from pointmvsnet_b200 import networks as ours_networks
        ref_networks.EdgeConv = ours_networks.EdgeConv
        ref_networks.EdgeConvNoC = ours_networks.EdgeConvNoC
        ref_networks.gather_knn = sys.modules["pointmvsnet.functions.gather_knn"].gather_knn
        return
    mapping = dict(hot)
    mapping.update(extra)
    for parent in ("pointmvsnet", "pointmvsnet.functions", "pointmvsnet.utils", "pointmvsnet.nn"):
        if parent not in sys.modules:
            stub = types.ModuleType(parent)
            stub.__path__ = []
            sys.modules[parent] = stub
    for ref_name, ours in mapping.items():
        mod = importlib.import_module(ours)
        sys.modules[ref_name] = mod
        parent, _, leaf = ref_name.rpartition(".")
        setattr(sys.modules[parent], leaf, mod)
    for parent in ("pointmvsnet.functions", "pointmvsnet.utils", "pointmvsnet.nn"):
        setattr(sys.modules["pointmvsnet"], parent.rpartition(".")[2], sys.modules[parent])
