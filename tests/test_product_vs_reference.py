"""Host-side containers and helpers of the product against the REAL reference classes.

What the reference classes returned is stored under tests/golden/reference/ (tests/helpers.py: reference_outputs; the
reference itself, loaded by path through oracle/refload.py, runs only to re-record it)."""
import json
import pickle

import numpy as np
import pandas as pd
import pytest
import torch

from megapose6d_b200 import pose_estimator as mine_pe
from megapose6d_b200 import tensor_collection as mine_tc
from megapose6d_b200.types import ObservationTensor as MineObs
from oracle import refload
from tests import helpers


def _frame(n, seed):
    rs = np.random.RandomState(seed)
    return pd.DataFrame(dict(label=[f"obj_{k}" for k in rs.randint(0, 3, n)], batch_im_id=rs.randint(0, 2, n),
                             score=rs.rand(n)), index=rs.permutation(n) + 10)


def _same(a, b):
    assert len(a) == len(b)
    pd.testing.assert_frame_equal(a.infos, b.infos)
    assert list(a.tensors.keys()) == list(b.tensors.keys())
    for k in a.tensors:
        assert torch.equal(a.tensors[k], b.tensors[k]), k


def _collection_steps(T, n, poses, boxes):
    """The same sequence of operations on module T's PandasTensorCollection: [(step name, collection)]."""
    a = T.PandasTensorCollection(infos=_frame(n, 1), poses=poses.clone(), bboxes=boxes.clone())
    steps = [("new", a)]                                   # index reset to 0..n-1 on construction
    for i, ids in enumerate(([2, 0, 5], torch.tensor([1, 1, 8]), np.array([3, 4]), [0])):
        steps.append((f"getitem{i}", a[ids]))
    extra = pd.DataFrame(dict(label=["obj_0", "obj_1", "obj_2"], diameter=[0.1, 0.2, 0.3]))
    steps.append(("merge", a.merge_df(extra, on="label")))
    steps.append(("concat", T.concatenate([a[[0, 1]], a[[5]]])))
    steps.append(("clone", a.clone()))
    a.register_tensor("extra", torch.arange(n))
    a.poses = a.poses * 2
    steps.append(("registered", a.clone()))
    a.delete_tensor("extra")
    steps.append(("pickled", pickle.loads(pickle.dumps(a))))
    steps.append(("double", a.double()))
    return steps


def test_pandas_tensor_collection_behaves_like_the_reference():
    n = 9
    g = torch.Generator().manual_seed(0)
    poses, boxes = torch.randn(n, 4, 4, generator=g), torch.randn(n, 4, generator=g)

    def reference():
        R = refload.load().tensor_collection
        d = {}
        for name, c in _collection_steps(R, n, poses, boxes):
            d.update(helpers.collection_arrays(name, c))
        d["device"] = str(R.PandasTensorCollection(infos=_frame(n, 1), poses=poses.clone()).device)
        d["len_empty_concat"] = len(R.concatenate([]))
        return d

    want = helpers.reference_outputs("pandas_tensor_collection", reference)
    for name, b in _collection_steps(mine_tc, n, poses, boxes):
        _same(helpers.StoredCollection(want, name), b)
    assert str(mine_tc.PandasTensorCollection(infos=_frame(n, 1), poses=poses.clone()).device) == str(want["device"])
    with pytest.raises(AttributeError):
        _ = mine_tc.PandasTensorCollection(infos=_frame(n, 1), poses=poses.clone()).not_a_tensor
    assert len(mine_tc.concatenate([])) == int(want["len_empty_concat"]) == 0


def test_observation_tensor_behaves_like_the_reference():
    rs = np.random.RandomState(3)
    rgb = rs.randint(0, 255, size=(12, 16, 3), dtype=np.uint8)
    depth = rs.rand(12, 16).astype(np.float32)
    K = np.array([[500.0, 0, 8], [0, 510, 6], [0, 0, 1]])
    rgb_b = torch.from_numpy(rs.randint(0, 255, size=(2, 3, 12, 16), dtype=np.uint8))
    dep_b = torch.from_numpy(rs.rand(2, 1, 12, 16).astype(np.float32))
    Kb = torch.from_numpy(np.stack([K, K])).float()

    def reference():
        RObs = refload.load().types.ObservationTensor
        out = {}
        for i, d in enumerate((None, depth)):
            a = RObs.from_numpy(rgb, d, K)
            out.update({f"{i}/images": a.images, f"{i}/K": a.K, f"{i}/batch_size": a.batch_size,
                        f"{i}/channel_dim": a.channel_dim, f"{i}/is_valid": a.is_valid()})
            if d is not None:
                out[f"{i}/depth"] = a.depth
        a = RObs.from_torch_batched(rgb_b, dep_b, Kb)
        out.update({"batched/images": a.images, "batched/K": a.K, "batched/channel_dim": a.channel_dim})
        try:
            RObs.from_torch_batched(rgb_b, dep_b[:, 0], Kb)
            out["bhw_depth_raises"] = False
        except RuntimeError:
            out["bhw_depth_raises"] = True
        return out

    want = helpers.reference_outputs("observation_tensor", reference)
    for i, d in enumerate((None, depth)):
        b = MineObs.from_numpy(rgb, d, K)
        assert torch.equal(want[f"{i}/images"], b.images) and torch.equal(want[f"{i}/K"], b.K)
        assert int(want[f"{i}/batch_size"]) == b.batch_size and int(want[f"{i}/channel_dim"]) == b.channel_dim
        assert bool(want[f"{i}/is_valid"]) == b.is_valid()
        if d is not None:
            assert torch.equal(want[f"{i}/depth"], b.depth)
    b = MineObs.from_torch_batched(rgb_b, dep_b, Kb)
    assert torch.equal(want["batched/images"], b.images) and torch.equal(want["batched/K"], b.K)
    assert int(want["batched/channel_dim"]) == b.channel_dim == 4
    # [B,H,W] depth: the reference drops the result of `depth.unsqueeze(1)` (inference/types.py:224-229) and raises; the
    # product accepts it as documented there
    assert bool(want["bhw_depth_raises"])
    assert torch.equal(MineObs.from_torch_batched(rgb_b, dep_b[:, 0], Kb).images, b.images)


FILTERS = (dict(labels=["obj_0", "obj_2"]), dict(one_instance_per_class=True),
           dict(labels=["obj_1"], one_instance_per_class=True))


def test_instance_ids_and_detection_filter_match_the_reference():
    n = 11

    def reference():
        ref = refload.load()
        R, U = ref.tensor_collection, ref.inference_utils
        out = {}
        for seed in range(4):
            boxes = torch.randn(n, 4, generator=torch.Generator().manual_seed(seed))
            a = U.add_instance_id(R.PandasTensorCollection(infos=_frame(n, seed), bboxes=boxes.clone()))
            out[f"{seed}/instance_id"] = a.infos["instance_id"].to_numpy()
            # (with this pandas the reference's groupby().apply() drops the grouping columns from `a.infos`; the product
            # keeps them, as the reference did with the pandas it was written for) -> give the reference filter the
            # complete frame
            b = mine_pe.add_instance_id(mine_tc.PandasTensorCollection(infos=_frame(n, seed), bboxes=boxes.clone()))
            a = R.PandasTensorCollection(infos=b.infos.copy(), bboxes=boxes.clone())
            for i, kwargs in enumerate(FILTERS):
                fa = U.filter_detections(a, **kwargs)
                out.update({f"{seed}/{i}/label": fa.infos["label"].to_numpy(), f"{seed}/{i}/score": fa.infos["score"].to_numpy(),
                            f"{seed}/{i}/bboxes": fa.bboxes})
        return out

    want = helpers.reference_outputs("instance_ids_and_filter", reference)
    for seed in range(4):
        boxes = torch.randn(n, 4, generator=torch.Generator().manual_seed(seed))
        b = mine_pe.add_instance_id(mine_tc.PandasTensorCollection(infos=_frame(n, seed), bboxes=boxes.clone()))
        assert want[f"{seed}/instance_id"].tolist() == b.infos["instance_id"].tolist()
        # an existing column is left alone
        assert mine_pe.add_instance_id(b).infos["instance_id"].tolist() == want[f"{seed}/instance_id"].tolist()
        for i, kwargs in enumerate(FILTERS):
            fb = mine_pe.filter_detections(b, **kwargs)
            assert list(want[f"{seed}/{i}/label"]) == fb.infos["label"].tolist()
            assert want[f"{seed}/{i}/score"].tolist() == fb.infos["score"].tolist()
            assert torch.equal(want[f"{seed}/{i}/bboxes"], fb.bboxes)


class _AttrDict(dict):
    """OmegaConf-like config for the reference function: attribute access, `in`, `del`, hasattr."""
    __getattr__ = lambda self, k: self[k] if k in self else (_ for _ in ()).throw(AttributeError(k))  # noqa: E731
    __setattr__ = dict.__setitem__
    __delattr__ = dict.__delitem__


def test_check_update_config_matches_the_reference():
    """training/pose_models_cfg.py:36-87 executed from the reference source (its module imports Panda3D, so only the
    function body is compiled) against load_model.check_update_config on legacy and current run configurations."""
    import logging
    import re

    from megapose6d_b200 import load_model

    cases = [
        dict(load_model.ZOO_CONFIGS["coarse-rgb-906902141"]),
        dict(load_model.ZOO_CONFIGS["refiner-rgbd-288182519"]),
        dict(input_strategy="input=obs+one_render", multiview_type="TCO", backbone_str="vanilla_resnet34"),
        dict(multiview_type="front_3views", n_views=4, backbone_str="vanilla_resnet34"),
        dict(multiview_type="front_5views", n_rendered_views=6, render_normals=True, depth_augmentation=True,
             depth_normalization_type="tCR_scale_clamp_center"),
    ]

    def reference():
        src = (refload.REF_ROOT / "training/pose_models_cfg.py").read_text()
        body = src[src.index("def check_update_config"):src.index("def create_model_pose")]
        body = re.sub(r"\(cfg: TrainingConfig\) -> TrainingConfig", "(cfg)", body)
        ns = dict(logger=logging.getLogger("ref"))
        exec(compile(body, "pose_models_cfg.py", "exec"), ns)
        return {str(i): helpers.json_array(dict(ns["check_update_config"](_AttrDict(case)))) for i, case in enumerate(cases)}

    stored = helpers.reference_outputs("check_update_config", reference)
    for i, case in enumerate(cases):
        want = json.loads(str(stored[str(i)]))
        got = load_model.check_update_config(load_model.Cfg(dict(case)))
        for key in ("is_coarse_compat", "n_rendered_views", "multiview_type", "predict_rendered_views_logits",
                    "remove_TCO_rendering", "predict_pose_update", "render_normals", "render_depth", "input_depth",
                    "renderer"):
            assert got[key] == want[key], (case, key, got[key], want[key])
        if "depth_normalization_type" in want:
            assert got["depth_normalization_type"] == want["depth_normalization_type"], case
        assert "n_views" not in got
