"""The DSB fixture cases: how each ``tests/golden/dsb_<case>.npz`` is laid out and how its call is rebuilt.

Shared by ``tests/golden/make_golden_dsb.py`` (which runs the reference on them) and the DSB tests (which run
``mu.prot.pp.dsb`` and ``oracle.dsb_ref`` on the stored inputs)."""
import json

import numpy as np
import scipy.sparse as sp

# name -> (cells, proteins, empty droplets, count dtype, layout, cells stored sparse, control columns, dsb kwargs)
CASES = {
    # seed 1: no fit of this case stops at a different round in float32 (reference) and float64 (here); such a
    # fit moves its cell's bgmean by up to the tolerance and, through the regression, every cell's output
    "f32": dict(n=1200, P=24, n_empty=5000, dtype="float32", layout="anndata", sparse=False, seed=1,
                kw=dict(random_state=42)),
    "f64": dict(n=800, P=130, n_empty=3000, dtype="float64", layout="anndata", sparse=True,
                kw=dict(scale_factor="mean_subtract", random_state=3)),
    "isotype": dict(n=600, P=20, n_empty=3000, dtype="int64", layout="anndata", sparse=False, controls=2,
                    kw=dict(isotype_controls=["ctrl0", "ctrl1", "ctrl_missing"], quantile_clipping=True,
                            random_state=5)),
    "rs": dict(n=500, P=16, n_empty=2000, dtype="float32", layout="anndata", sparse=True,
               kw=dict(random_state=["RandomState", 7])),
    "nodenoise": dict(n=400, P=30, n_empty=2000, dtype="float32", layout="anndata", sparse=False,
                      kw=dict(denoise_counts=False, add_layer=True)),
    "mudata": dict(n=300, P=12, n_empty=1500, dtype="float64", layout="mudata_none", sparse=True,
                   kw=dict(empty_counts_range=[1.5, 2.5], cell_counts_range=[3.0, 4.0], random_state=11)),
    "mudata_raw": dict(n=300, P=12, n_empty=1500, dtype="float32", layout="mudata_raw", sparse=True,
                       kw=dict(empty_counts_range=[1.5, 2.5], random_state=13)),
}
N_JUNK = 200        # barcodes below both count ranges in the MuData layouts
N_OVERLAP = 5       # cells whose RNA count falls in the empty range (mudata_raw: "Dropping ..." warning)


def make_inputs(name, seed=None):
    """Arrays of one case (what the npz stores besides the outputs)."""
    from oracle.dsb_ref import synth_citeseq
    c = CASES[name]
    seed = c.get("seed", 0) if seed is None else seed
    n, P, m = c["n"], c["P"], c["n_empty"]
    dt = np.dtype(c["dtype"])
    cells, empty = synth_citeseq(n, m, P, seed=seed + sum(map(ord, name)),
                                 dtype=np.float64 if dt.kind != "f" else dt)
    cells, empty = cells.astype(dt), empty.astype(dt)
    nc = c.get("controls", 0)
    var = np.array([f"ctrl{j}" for j in range(nc)] + [f"p{j}" for j in range(nc, P)])
    out = {"var_names": var, "cells": cells, "empty": empty}
    if c["layout"] != "anndata":
        rng = np.random.default_rng(seed + 1)
        junk = sp.csr_matrix((rng.poisson(0.3, (N_JUNK, P)) > 0).astype(dt))
        prot = sp.vstack([sp.csr_matrix(cells), empty, junk], format="csr")
        lo = {"cell": 3.0, "empty": 1.5, "junk": 0.0}
        kinds = ["cell"] * n + ["empty"] * m + ["junk"] * N_JUNK
        if c["layout"] == "mudata_raw":
            kinds[:N_OVERLAP] = ["empty"] * N_OVERLAP
        umi = np.floor(10 ** np.array([lo[k] + 0.9 * rng.random() for k in kinds]))
        genes = rng.integers(0, 40, len(kinds))
        out["rna"] = sp.csr_matrix((umi, (np.arange(len(kinds)), genes)), shape=(len(kinds), 40))
        out["prot"] = prot
    return out


def pack(arrays):
    """npz-ready dict: CSR matrices split into parts."""
    z = {}
    for k, v in arrays.items():
        if sp.issparse(v):
            v = sp.csr_matrix(v)
            z.update({f"{k}__data": v.data, f"{k}__indices": v.indices.astype(np.int32),
                      f"{k}__indptr": v.indptr.astype(np.int64), f"{k}__shape": np.asarray(v.shape)})
        else:
            z[k] = np.asarray(v)
    return z


def unpack(z, key):
    if f"{key}__data" in z:
        return sp.csr_matrix((z[f"{key}__data"], z[f"{key}__indices"], z[f"{key}__indptr"]),
                             shape=tuple(int(s) for s in z[f"{key}__shape"]))
    return z[key]


def kwargs(name, z=None):
    kw = json.loads(str(z["kwargs"])) if z is not None else json.loads(json.dumps(CASES[name]["kw"]))
    rs = kw.get("random_state")
    if isinstance(rs, list):
        kw["random_state"] = np.random.RandomState(rs[1])
    for k in ("empty_counts_range", "cell_counts_range", "quantile_clip"):
        if k in kw:
            kw[k] = tuple(kw[k])
    return kw


def build_call(name, z, AnnData, MuData):
    """(data, data_raw, kwargs) of one case, freshly built from its stored inputs with the given containers."""
    c = CASES[name]
    var = [str(v) for v in z["var_names"]]
    cells = unpack(z, "cells")
    if not c["sparse"] and sp.issparse(cells):
        cells = cells.toarray()
    kw = kwargs(name, z)
    n = cells.shape[0]
    if c["layout"] == "anndata":
        empty = unpack(z, "empty")
        data = AnnData(cells.copy(), obs=[f"cell{i}" for i in range(n)], var=var)
        raw = AnnData(empty.copy(), obs=[f"empty{i}" for i in range(empty.shape[0])], var=var)
        return data, raw, kw
    rna, prot = unpack(z, "rna"), unpack(z, "prot")
    bcs = [f"bc{i}" for i in range(prot.shape[0])]
    raw = MuData({"rna": AnnData(rna.copy(), obs=bcs, var=[f"g{j}" for j in range(rna.shape[1])]),
                  "prot": AnnData(prot.copy(), obs=bcs, var=var)})
    if c["layout"] == "mudata_none":
        return raw, None, kw
    return AnnData(cells.copy(), obs=bcs[:n], var=var), raw, kw


def ref_arguments(name, z):
    """(cells, empty droplets, dsb_ref keyword arguments) of one case: the droplet selection of the reference's
    container branches (preproc.py:66-160) done by hand, so that ``oracle.dsb_ref`` sees the same matrices."""
    c = CASES[name]
    kw = kwargs(name, z)
    if c["layout"] == "anndata":
        cells, empty = unpack(z, "cells"), unpack(z, "empty")
    else:
        prot = unpack(z, "prot")
        lu = np.log10(np.asarray(unpack(z, "rna").sum(axis=1)).ravel() + 1)
        e0, e1 = kw["empty_counts_range"]
        emp = np.where((lu >= e0) & (lu < e1))[0]
        if c["layout"] == "mudata_none":
            c0, c1 = kw["cell_counts_range"]
            cells = prot[np.where((lu >= c0) & (lu < c1))[0]]
        else:
            cells = unpack(z, "cells")
            emp = emp[emp >= c["n"]]
        empty = prot[emp]
    var = [str(v) for v in z["var_names"]]
    ctrl = kw.get("isotype_controls")
    return cells, empty, dict(
        pseudocount=kw.get("pseudocount", 10), denoise_counts=kw.get("denoise_counts", True),
        ctrl_idx=None if ctrl is None else np.where(np.isin(var, list(ctrl)))[0],
        scale_factor=kw.get("scale_factor", "standardize"),
        quantile_clip=kw.get("quantile_clip", (0.001, 0.9995)) if kw.get("quantile_clipping") else None,
        random_state=kw.get("random_state"))


def result_of(name, data, data_raw, returned):
    """The normalised matrix the call left behind (and the observation names it belongs to)."""
    c = CASES[name]
    if c["layout"] == "mudata_none":
        cells = returned.mod["prot"]
    else:
        cells = data if data_raw is not None and not hasattr(data, "mod") else data.mod["prot"]
    X = cells.layers["dsb"] if c["kw"].get("add_layer") else cells.X
    return np.asarray(X), np.asarray([str(s) for s in cells.obs_names])
