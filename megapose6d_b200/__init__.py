"""H100-native render-and-compare pose engine with the MegaPose inference API.

Public surface (mirrors the reference's import points):
    PoseEstimator, PosePredictor, BatchRenderer (alias Panda3dBatchRenderer), ObservationTensor,
    PandasTensorCollection, RigidObject, RigidObjectDataset, NAMED_MODELS, load_named_model, TeaserppRefiner.
The CUDA library is loaded lazily on first use; see megapose6d_b200/_abi.py and include/mpx.h.
"""
__all__ = [
    "PoseEstimator", "PosePredictor", "BatchRenderer", "Panda3dBatchRenderer", "ObservationTensor",
    "PandasTensorCollection", "RigidObject", "RigidObjectDataset", "NAMED_MODELS", "load_named_model",
    "TeaserppRefiner",
]


def __getattr__(name):
    import importlib

    table = {
        "PoseEstimator": ".pose_estimator", "PosePredictor": ".pose_predictor", "BatchRenderer": ".renderer",
        "Panda3dBatchRenderer": ".renderer", "ObservationTensor": ".types", "PandasTensorCollection": ".tensor_collection",
        "RigidObject": ".object_dataset", "RigidObjectDataset": ".object_dataset", "NAMED_MODELS": ".load_model",
        "load_named_model": ".load_model", "TeaserppRefiner": ".teaserpp_refiner",
    }
    if name in table:
        return getattr(importlib.import_module(table[name], __name__), name)
    raise AttributeError(name)
