"""Generate tests/golden/validate_metrics.npz from the UNMODIFIED reference accumulation code:
unidepth/datasets/base_dataset.py's BaseDataset (accumulate_metrics, prepare_depth_eval, prepare_points_eval,
add_points, accumulate_metrics_depth, accumulate_metrics_3d, get_evaluation), with the reference's eval_depth / eval_3d,
camera classes and the KNN CPU extension (compiled into oracle/_ref/ as make_golden_eval.py does).

unidepth.datasets' package __init__ imports every dataset (and h5py), so base_dataset.py is loaded by path under a stub
`unidepth.datasets` package whose `pipelines` module is empty; everything else it imports comes from the reference tree
through oracle/ref_shims.  The methods run on an instance created without BaseDataset.__init__ (which reads split files),
with min_depth / max_depth from oracle/validate_oracle.py and empty stores, over the seeded batches of
validate_oracle.batches.  Stored: every metrics_store tensor before get_evaluation (`store/{eval_type}/{name}`), the
metrics_count tensors (`count/{eval_type}`), and get_evaluation's dict (`eval/{key}`).

Run on a machine with the reference tree:   python oracle/make_golden_validate.py [/path/to/reference]
TEST INFRASTRUCTURE ONLY.
"""
import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
sys.path[:0] = [REF, os.path.join(HERE, "ref_shims"), HERE]


def load_base_dataset():
    import unidepth  # noqa: F401
    pkg = types.ModuleType("unidepth.datasets")
    pkg.__path__ = [os.path.join(REF, "unidepth", "datasets")]
    sys.modules["unidepth.datasets"] = pkg
    sys.modules["unidepth.datasets.pipelines"] = types.ModuleType("unidepth.datasets.pipelines")
    path = os.path.join(REF, "unidepth", "datasets", "base_dataset.py")
    spec = importlib.util.spec_from_file_location("unidepth.datasets.base_dataset", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod.BaseDataset


def main():
    warnings.simplefilter("ignore")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    from make_golden_eval import load_knn
    load_knn()
    import validate_oracle as V
    import unidepth.utils.camera as C
    BaseDataset = load_base_dataset()

    class Stub(BaseDataset):
        pass

    ds = object.__new__(Stub)
    ds.min_depth, ds.max_depth = V.MIN_DEPTH, V.MAX_DEPTH
    ds.metrics_store, ds.metrics_count = {}, {}
    for inputs, preds, kf in V.batches(C):
        ds.accumulate_metrics(inputs=inputs, preds=preds, keyframe_idx=kf)
    out = {}
    for eval_type, store in ds.metrics_store.items():
        for name, v in store.items():
            out[f"store/{eval_type}/{name}"] = v.numpy()
        out[f"count/{eval_type}"] = ds.metrics_count[eval_type].numpy()
    ev = ds.get_evaluation()
    for k, v in ev.items():
        out[f"eval/{k}"] = np.float64(v)
    out["eval_keys"] = np.array(list(ev))
    print({k: v for k, v in ev.items()})
    path = os.path.join(ROOT, "tests", "golden", "validate_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
