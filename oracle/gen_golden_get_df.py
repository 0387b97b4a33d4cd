"""Generates tests/golden/ref_get_df.npz by RUNNING THE REFERENCE's preprocess.get_df() (needs pandas, pyarrow, joblib,
tqdm and a checkout of handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE).

For every fixture, synthetic.make_raw_tables(seed, dotted_rpcid) is written to data/MSCallGraph/*.csv and
data/MSResource/*.csv of a temporary working directory without processed/*.csv, so get_df() (:191-266) takes its
raw-data branch.  Stored, per fixture prefix:
  callgraph_files / resource_files   the os.listdir order get_df() concatenated the files in (the tests pass it on)
  df_<column>, df_index              processed_df column by column (:263 endTimestamp included) and its index
  res_<column>                       processed_resource_df column by column
  dtype_df_<column>, dtype_res_<column>  the pandas dtype of every column
The CSV text is regenerated from the seed by the tests (make_raw_tables is deterministic).  The reference numbers
microservices in Python set order, so the generator runs under PYTHONHASHSEED=0 (re-executing itself if needed) and
writes the archive with fixed zip timestamps: regenerating gives the same file byte for byte.
Usage:  PERT_GNN_REFERENCE=<checkout> python oracle/gen_golden_get_df.py
"""
import importlib.util
import os
import sys
import tempfile
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pert_gnn_kdd23_b200.synthetic import make_raw_tables  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_get_df.npz")
FIXTURES = {"numeric": (0, False), "dotted": (1, True)}       # prefix -> (seed, dotted_rpcid)


def write_fixture(work, seed, dotted):
    d = make_raw_tables(seed, dotted_rpcid=dotted)
    for sub, files in (("MSCallGraph", d["callgraph"]), ("MSResource", d["resource"])):
        os.makedirs(os.path.join(work, "data", sub))
        for name, text in files.items():
            with open(os.path.join(work, "data", sub, name), "w") as f:
                f.write(text)


def _column(s):
    """A frame column as a plain numpy array (object columns of ints / floats converted)."""
    a = s.to_numpy()
    if a.dtype == object:
        a = np.array(a.tolist())
    return a


def savez_fixed(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member, so equal arrays give an equal file."""
    import io
    import zipfile

    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    if os.environ.get("PYTHONHASHSEED") != "0":
        os.execve(sys.executable, [sys.executable] + sys.argv, dict(os.environ, PYTHONHASHSEED="0"))
    import pandas as pd

    pd.set_option("future.infer_string", False)          # map_consecutive_ids writes int codes into the Series
    warnings.simplefilter("ignore")
    ref = os.environ["PERT_GNN_REFERENCE"]
    out = {}
    cwd = os.getcwd()
    for fx, (seed, dotted) in FIXTURES.items():
        with tempfile.TemporaryDirectory() as work:
            write_fixture(work, seed, dotted)
            os.makedirs(os.path.join(work, "processed"))
            os.chdir(work)
            sys.path.insert(0, ref)
            try:
                spec = importlib.util.spec_from_file_location("_ref_preprocess", os.path.join(ref, "preprocess.py"))
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                df, res = mod.get_df()
                out[f"{fx}_callgraph_files"] = np.array([f for f in os.listdir("data/MSCallGraph")
                                                         if f.endswith(".csv")])
                out[f"{fx}_resource_files"] = np.array([f for f in os.listdir("data/MSResource")
                                                        if f.endswith(".csv")])
            finally:
                os.chdir(cwd)
                sys.path.remove(ref)
        out[f"{fx}_seed"] = np.int64(seed)
        out[f"{fx}_dotted"] = np.bool_(dotted)
        out[f"{fx}_df_index"] = df.index.to_numpy().astype(np.int64)
        for tag, frame in (("df", df), ("res", res)):
            for c in frame.columns:
                out[f"{fx}_{tag}_{c}"] = _column(frame[c])
                out[f"{fx}_dtype_{tag}_{c}"] = np.array(str(frame[c].dtype))
        print(fx, len(df), "rows,", df.traceid.nunique(), "traces,", len(res), "resource rows")
    savez_fixed(OUT, out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
