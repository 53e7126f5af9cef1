"""Readers of the four datasets that have a config (AdaQP/helper/dataset.py, helper/partition.py:10-60),
numpy / scipy only.  They read files already under `raw_dir` and never download; a missing file raises
FileNotFoundError naming the expected path and where the reference gets it.

Each reader returns one `GlobalGraph`: a symmetric CSR with exactly one self-loop per node and no
multi-edges (helper/partition.py:57-60: remove self-loops, add one per node; parallel edges collapse as in
the rest of the ingest), float32 features, labels (int64 [N], or float32 [N, C] for multilabel datasets) and
train / val / test masks.  Global degrees are the CSR row lengths.  A graph that is not symmetric is refused
with NotImplementedError, as the Trainer refuses directed partitions (DESIGN.md section 6).
"""
from __future__ import annotations

import gzip
import json
import os
from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp


@dataclass
class GlobalGraph:
    name: str
    indptr: np.ndarray          # int64 [N + 1]
    indices: np.ndarray         # int32, sorted within rows, self-loop included
    feat: np.ndarray            # float32 [N, F]
    label: np.ndarray           # int64 [N] or float32 [N, C]
    train_mask: np.ndarray
    val_mask: np.ndarray
    test_mask: np.ndarray
    n_collapsed: int = 0        # parallel (non-self) directed edges merged into one

    @property
    def num_nodes(self) -> int:
        return self.indptr.size - 1

    @property
    def degrees(self) -> np.ndarray:
        return np.diff(self.indptr).astype(np.int64)

    def permuted(self, perm: np.ndarray) -> "GlobalGraph":
        """The same graph with node i of the result = node perm[i] of this one."""
        A = sp.csr_matrix((np.ones(self.indices.size, np.int8), self.indices, self.indptr))[perm][:, perm].tocsr()
        A.sort_indices()
        return GlobalGraph(name=self.name, indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32),
                           feat=self.feat[perm], label=self.label[perm], train_mask=self.train_mask[perm],
                           val_mask=self.val_mask[perm], test_mask=self.test_mask[perm], n_collapsed=self.n_collapsed)


SOURCES = {
    "ogbn-products": "the OGB download of ogbn-products (ogb.nodeproppred.DglNodePropPredDataset, "
                     "helper/partition.py:14), unpacked as ogbn_products/",
    "reddit": "DGL's RedditDataset download (dgl.data.RedditDataset, helper/partition.py:48)",
    "yelp": "the GraphSAINT Yelp files the reference's load_yelp reads (helper/dataset.py:123-161)",
    "amazonProducts": "the GraphSAINT AmazonProducts files the reference downloads (helper/dataset.py:55-72)",
}


def _need(path: str, dataset: str) -> str:
    if not os.path.exists(path):
        raise FileNotFoundError(f"{dataset}: expected {path}; get it from {SOURCES[dataset]}. "
                                f"Nothing is downloaded here.")
    return path


def _read_csv_gz(path: str, dtype, cols: int) -> np.ndarray:
    with gzip.open(path, "rb") as f:
        text = f.read().replace(b",", b" ").decode("ascii")
    return np.array(text.split(), dtype=dtype).reshape(-1, cols) if cols > 1 else np.array(text.split(), dtype=dtype)


def _mask(n: int, idx) -> np.ndarray:
    m = np.zeros(n, bool)
    m[np.asarray(idx, np.int64)] = True
    return m


def finish_graph(name: str, src, dst, n: int, feat, label, train, val, test) -> GlobalGraph:
    """Common preprocessing of helper/partition.py:57-60 on an edge list (src -> dst)."""
    src = np.asarray(src, np.int64)
    dst = np.asarray(dst, np.int64)
    keep = src != dst
    src, dst = src[keep], dst[keep]
    A = sp.csr_matrix((np.ones(src.size, np.int32), (dst, src)), shape=(n, n))
    A.sum_duplicates()
    n_collapsed = int(src.size - A.nnz)
    A.data[:] = 1
    if (A != A.T).nnz:
        raise NotImplementedError(f"{name}: the graph is not symmetric; directed graphs are not supported "
                                  f"(in_degrees != out_degrees, DESIGN.md section 6)")
    A = (A + sp.identity(n, np.int32, format="csr")).tocsr()
    A.sort_indices()
    return GlobalGraph(name=name, indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32),
                       feat=np.ascontiguousarray(feat, np.float32), label=label, train_mask=train, val_mask=val,
                       test_mask=test, n_collapsed=n_collapsed)


def load_ogbn_products(raw_dir: str) -> GlobalGraph:
    """OGB raw layout; OGB adds the inverse edges for products (add_inverse_edge); labels[:, 0]; masks from the
    sales_ranking split (helper/partition.py:10-30)."""
    d, name = os.path.join(raw_dir, "ogbn_products"), "ogbn-products"
    edge = _read_csv_gz(_need(os.path.join(d, "raw", "edge.csv.gz"), name), np.int64, 2)
    feat_path = _need(os.path.join(d, "raw", "node-feat.csv.gz"), name)
    label = _read_csv_gz(_need(os.path.join(d, "raw", "node-label.csv.gz"), name), np.int64, 1)
    split = [_read_csv_gz(_need(os.path.join(d, "split", "sales_ranking", f"{s}.csv.gz"), name), np.int64, 1)
             for s in ("train", "valid", "test")]
    n = label.size
    feat = _read_csv_gz(feat_path, np.float32, 1).reshape(n, -1)
    src = np.concatenate([edge[:, 0], edge[:, 1]])
    dst = np.concatenate([edge[:, 1], edge[:, 0]])
    return finish_graph(name, src, dst, n, feat, label.astype(np.int64), *(_mask(n, s) for s in split))


def load_reddit(raw_dir: str) -> GlobalGraph:
    """DGL 0.9 RedditDataset layout: reddit_data.npz (feature, label, node_types) and reddit_graph.npz (scipy
    sparse); masks are node_types == 1 / 2 / 3."""
    d, name = os.path.join(raw_dir, "reddit"), "reddit"
    data = np.load(_need(os.path.join(d, "reddit_data.npz"), name))
    A = sp.load_npz(_need(os.path.join(d, "reddit_graph.npz"), name)).tocoo()
    nt = data["node_types"]
    n = nt.size
    return finish_graph(name, A.row, A.col, n, data["feature"], data["label"].astype(np.int64),
                        nt == 1, nt == 2, nt == 3)


def _saint_common(raw_dir: str, name: str):
    d = os.path.join(raw_dir, name)
    paths = {f: _need(os.path.join(d, f), name) for f in ("adj_full.npz", "feats.npy", "class_map.json", "role.json")}
    with open(paths["class_map.json"]) as f:
        class_map = json.load(f)
    with open(paths["role.json"]) as f:
        role = json.load(f)
    return paths, class_map, role


def _labels(values) -> np.ndarray:
    arr = np.asarray(values)
    return arr.astype(np.float32) if arr.ndim == 2 else arr.astype(np.int64)


def load_yelp(raw_dir: str) -> GlobalGraph:
    """helper/dataset.py:123-161: labels in class_map file order; features standardised with the mean and the
    population std of the train rows (a zero-std column keeps scale 1, as sklearn's StandardScaler)."""
    paths, class_map, role = _saint_common(raw_dir, "yelp")
    A = sp.load_npz(paths["adj_full.npz"]).tocoo()
    feats = np.load(paths["feats.npy"])
    n = feats.shape[0]
    train, val, test = (_mask(n, role[k]) for k in ("tr", "va", "te"))
    x = feats.astype(np.float64)
    mean = x[train].mean(0)
    std = x[train].std(0)
    std[std == 0] = 1.0
    feat = ((x - mean) / std).astype(np.float32)
    return finish_graph("yelp", A.row, A.col, n, feat, _labels(list(class_map.values())), train, val, test)


def load_amazon_products(raw_dir: str) -> GlobalGraph:
    """helper/dataset.py:74-103: row int(key) of the labels is class_map[key].  The reference's
    dgl.reorder_graph(rcmk) only permutes ids before the partitioner relabels them; it is not restated."""
    paths, class_map, role = _saint_common(raw_dir, "amazonProducts")
    f = np.load(paths["adj_full.npz"])
    A = sp.csr_matrix((f["data"], f["indices"], f["indptr"]), tuple(f["shape"])).tocoo()
    feats = np.load(paths["feats.npy"]).astype(np.float32)
    n = feats.shape[0]
    keys = np.fromiter((int(k) for k in class_map), np.int64, len(class_map))
    vals = _labels(list(class_map.values()))
    label = np.zeros((n,) + vals.shape[1:], vals.dtype)
    label[keys] = vals
    train, val, test = (_mask(n, role[k]) for k in ("tr", "va", "te"))
    return finish_graph("amazonProducts", A.row, A.col, n, feats, label, train, val, test)


READERS = {"ogbn-products": load_ogbn_products, "reddit": load_reddit, "yelp": load_yelp,
           "amazonProducts": load_amazon_products}


def load_dataset(dataset: str, raw_dir: str) -> GlobalGraph:
    if dataset not in READERS:
        raise ValueError(f"no such dataset: {dataset} (readers: {sorted(READERS)})")
    return READERS[dataset](raw_dir)
