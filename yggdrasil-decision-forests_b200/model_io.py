"""YDF model directory I/O for the trained forest.

Writing goes through the native writer (csrc/ygg_model_io.cc, `ygg_model_write_ydf`); this module
only serialises the DataSpecification (it owns column names / boundaries) and provides a small
proto2 wire reader used by the tests to read a model directory back — ours or the reference's
(model/gradient_boosted_trees/gradient_boosted_trees.cc:111-139, utils/blob_sequence.h:121-149).
"""
import ctypes as C
import os
import struct
from typing import List

import numpy as np

from . import _capi


# ---- minimal proto2 wire encoder / decoder -------------------------------------------------------
def _varint(v: int) -> bytes:
    v &= (1 << 64) - 1
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _key(field, wire):
    return _varint(field << 3 | wire)


def pb_int(field, v):
    return _key(field, 0) + _varint(int(v))


def pb_f32(field, v):
    return _key(field, 5) + struct.pack("<f", v)


def pb_f64(field, v):
    return _key(field, 1) + struct.pack("<d", v)


def pb_bytes(field, b):
    if isinstance(b, str):
        b = b.encode()
    return _key(field, 2) + _varint(len(b)) + b


def pb_decode(b: bytes):
    """-> list of (field, wire_type, value); nested messages stay bytes."""
    i, out = 0, []
    while i < len(b):
        k = 0
        s = 0
        while True:
            c = b[i]
            i += 1
            k |= (c & 0x7F) << s
            s += 7
            if not c & 0x80:
                break
        f, w = k >> 3, k & 7
        if w == 0:
            v = 0
            s = 0
            while True:
                c = b[i]
                i += 1
                v |= (c & 0x7F) << s
                s += 7
                if not c & 0x80:
                    break
            out.append((f, w, v))
        elif w == 1:
            out.append((f, w, struct.unpack("<d", b[i:i + 8])[0]))
            i += 8
        elif w == 5:
            out.append((f, w, struct.unpack("<f", b[i:i + 4])[0]))
            i += 4
        elif w == 2:
            n = 0
            s = 0
            while True:
                c = b[i]
                i += 1
                n |= (c & 0x7F) << s
                s += 7
                if not c & 0x80:
                    break
            out.append((f, w, b[i:i + n]))
            i += n
        else:
            raise ValueError(f"unsupported wire type {w}")
    return out


# ---- DataSpecification (dataset/data_spec.proto) --------------------------------------------------
def encode_data_spec(spec) -> (bytes, int, List[int]):
    """Column 0 is the label, columns 1.. the features.  Returns (bytes, label_col_idx, feature_col_idx)."""
    cols = []
    if spec.task == "CLASSIFICATION":
        cat = pb_int(1, 2) + pb_int(2, len(spec.label_classes) + 1)  # most_frequent_value, number_of_unique_values
        items = [("<OOD>", 0)] + [(str(c), i + 1) for i, c in enumerate(spec.label_classes)]
        for name, idx in items:
            vv = pb_int(1, idx) + pb_int(2, 0)  # VocabValue{index, count}
            cat += pb_bytes(7, pb_bytes(1, name) + pb_bytes(2, vv))  # map<string, VocabValue> entry
        cols.append(pb_int(1, 4) + pb_bytes(2, spec.label) + pb_int(3, 0) + pb_bytes(6, cat))  # CATEGORICAL
    else:
        num = pb_f64(1, spec.label_mean) + pb_f32(2, spec.label_min) + pb_f32(3, spec.label_max) + \
            pb_f64(4, spec.label_sd)
        cols.append(pb_int(1, 1) + pb_bytes(2, spec.label) + pb_int(3, 0) + pb_bytes(5, num))  # NUMERICAL
    for c in spec.columns:
        if getattr(c, "vocabulary", None) is not None:
            cat = pb_int(1, c.na_bin) + pb_int(2, c.num_bins)  # most_frequent_value, number_of_unique_values
            for idx, (key, count) in enumerate(zip(c.vocabulary, c.counts)):
                vv = pb_int(1, idx) + pb_int(2, count)
                cat += pb_bytes(7, pb_bytes(1, key) + pb_bytes(2, vv))
            cols.append(pb_int(1, 4) + pb_bytes(2, c.name) + pb_int(3, 0) + pb_bytes(6, cat) +
                        pb_int(7, c.num_missing))  # CATEGORICAL
            continue
        if getattr(c, "feature_type", None) == _capi.FEATURE_NUMERICAL:   # a presorted column: NUMERICAL, Higher splits
            num = pb_f64(1, c.mean) + pb_f32(2, c.min_value) + pb_f32(3, c.max_value)
            cols.append(pb_int(1, 1) + pb_bytes(2, c.name) + pb_int(3, 0) + pb_bytes(5, num) + pb_int(7, c.num_missing))
            continue
        num = pb_f64(1, c.mean)
        if len(c.boundaries):
            num += pb_f32(2, float(c.boundaries[0])) + pb_f32(3, float(c.boundaries[-1]))
        disc = pb_bytes(1, np.asarray(c.boundaries, dtype="<f4").tobytes())  # packed repeated float
        # maximum_num_bins: the budget asked for above 256 bins; else 255 for the discretized and byte lossless columns
        # and a wide lossless column's own bucket count
        budget = getattr(c, "maximum_num_bins", None)
        if budget is None:
            budget = max(255, len(c.boundaries) + 1) if c.num_bins > 256 else 255
        disc += pb_int(3, budget) + pb_int(4, 3)
        col = pb_int(1, 9) + pb_bytes(2, c.name) + pb_int(3, 0) + pb_bytes(5, num)  # DISCRETIZED_NUMERICAL
        col += pb_int(7, c.num_missing) + pb_bytes(8, disc)
        cols.append(col)
    out = b"".join(pb_bytes(1, c) for c in cols) + pb_int(2, spec.num_rows)
    return out, 0, list(range(1, len(spec.columns) + 1))


class ModelDesc(C.Structure):
    _fields_ = [
        ("directory", C.c_char_p), ("task", C.c_int32), ("loss", C.c_int32),
        ("use_hessian_gain", C.c_int32), ("initial_prediction", C.c_float),
        ("num_trees", C.c_int32), ("trees", C.c_void_p), ("tree_offsets", C.POINTER(C.c_int64)),
        ("num_features", C.c_int32), ("feature_col_idx", C.POINTER(C.c_int32)),
        ("label_col_idx", C.c_int32), ("data_spec_pb", C.c_char_p), ("data_spec_len", C.c_int64),
        ("train_loss", C.POINTER(C.c_float)), ("train_secondary", C.POINTER(C.c_float)),
        ("num_log_entries", C.c_int32), ("valid_loss", C.POINTER(C.c_float)),
        ("valid_secondary", C.POINTER(C.c_float)), ("has_validation_loss", C.c_int32),
        ("validation_loss", C.c_float), ("early_stopping_triggered", C.c_int32),
        ("num_trees_per_iter", C.c_int32), ("feature_num_values", C.POINTER(C.c_int32)),
        ("node_set_offset", C.POINTER(C.c_int64)), ("cat_set_words", C.POINTER(C.c_uint32)),
    ]


def save_ydf_model(model, path: str):
    spec_pb, label_idx, feat_idx = encode_data_spec(model.data_spec)
    trees = np.concatenate(model.trees) if model.trees else np.zeros(0, dtype=_capi.NODE_DTYPE)
    trees = np.ascontiguousarray(trees)
    offs = np.zeros(len(model.trees) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(t) for t in model.trees])
    fidx = np.asarray(feat_idx, dtype=np.int32)
    loss = np.asarray([l["loss"] for l in model.training_logs], dtype=np.float32)
    sec = np.asarray([l["secondary"] for l in model.training_logs], dtype=np.float32)
    d = ModelDesc()
    d.directory = os.fsencode(path)
    d.task = 1 if model.task() == "CLASSIFICATION" else 2
    d.loss = {"BINOMIAL_LOG_LIKELIHOOD": 0, "SQUARED_ERROR": 1, "MULTINOMIAL_LOG_LIKELIHOOD": 2}[model.loss]
    d.num_trees_per_iter = model.num_trees_per_iter()
    d.use_hessian_gain = int(model.config.get("use_hessian_gain", 0))
    d.initial_prediction = model.initial_prediction
    d.num_trees = len(model.trees)
    d.trees = trees.ctypes.data
    d.tree_offsets = offs.ctypes.data_as(C.POINTER(C.c_int64))
    d.num_features = len(fidx)
    d.feature_col_idx = fidx.ctypes.data_as(C.POINTER(C.c_int32))
    d.label_col_idx = label_idx
    d.data_spec_pb = spec_pb
    d.data_spec_len = len(spec_pb)
    d.num_log_entries = len(model.training_logs)
    d.train_loss = loss.ctypes.data_as(C.POINTER(C.c_float)) if len(loss) else None
    d.train_secondary = sec.ctypes.data_as(C.POINTER(C.c_float)) if len(sec) else None
    vl = np.asarray([l["validation_loss"] for l in model.training_logs if "validation_loss" in l], dtype=np.float32)
    vs = np.asarray([l["validation_secondary"] for l in model.training_logs if "validation_loss" in l], dtype=np.float32)
    if len(vl) == len(model.training_logs) and len(vl):
        d.valid_loss = vl.ctypes.data_as(C.POINTER(C.c_float))
        d.valid_secondary = vs.ctypes.data_as(C.POINTER(C.c_float))
    if getattr(model, "validation_loss", None) is not None:
        d.has_validation_loss, d.validation_loss = 1, float(model.validation_loss)
        d.early_stopping_triggered = int(bool(getattr(model, "early_stopping_triggered", False)))
    nvals = np.asarray([getattr(c, "num_bins", 0) for c in model.data_spec.columns], dtype=np.int32)
    d.feature_num_values = nvals.ctypes.data_as(C.POINTER(C.c_int32))
    # positive sets of the splits on wide categorical columns
    sets = getattr(model, "category_sets", None) or [{} for _ in model.trees]
    set_off = np.full(len(trees), -1, dtype=np.int64)
    chunks, used = [], 0
    for t, tree_sets in enumerate(sets):
        for node, words in sorted(tree_sets.items()):
            set_off[offs[t] + node] = used
            chunks.append(np.asarray(words, dtype=np.uint32))
            used += len(chunks[-1])
    words_all = np.ascontiguousarray(np.concatenate(chunks) if chunks else np.zeros(1, np.uint32))
    if chunks:
        d.node_set_offset = set_off.ctypes.data_as(C.POINTER(C.c_int64))
        d.cat_set_words = words_all.ctypes.data_as(C.POINTER(C.c_uint32))
    st = _capi.lib().ygg_model_write_ydf(C.byref(d))
    if st != 0:
        raise _capi.YggError(st, f"could not write the model to {path}")


# ---- reader (tests) ---------------------------------------------------------------------------------
def read_blob_sequence(path):
    """utils/blob_sequence.{h,cc}: 8-byte file header ("BS", u16 version, u8 compression), then records
    [u32 length][bytes]; with compression = GZIP (version >= 1) everything after the header is one gzip stream."""
    b = open(path, "rb").read()
    if b[:2] != b"BS":
        raise ValueError("not a blob sequence")
    version = struct.unpack("<H", b[2:4])[0]
    body = b[8:]
    if version >= 1 and b[4] == 1:
        import zlib
        body = zlib.decompress(body, wbits=31)
    elif version >= 1 and b[4] != 0:
        raise ValueError(f"unknown blob sequence compression {b[4]}")
    i, out = 0, []
    while i < len(body):
        n = struct.unpack("<I", body[i:i + 4])[0]
        out.append(body[i + 4:i + 4 + n])
        i += 4 + n
    return out


def _one(fields, f, default=None):
    for ff, _, v in fields:
        if ff == f:
            return v
    return default


def decode_node(rec: bytes) -> dict:
    """decision_tree::proto::Node -> dict (regression output + discretized/higher condition)."""
    f = pb_decode(rec)
    out = {"n": _one(f, 4)}
    reg = _one(f, 2)
    if reg is not None:
        r = pb_decode(reg)
        out["top_value"] = _one(r, 1)
        dist = _one(r, 2)
        if dist is not None:
            dd = pb_decode(dist)
            out["distribution"] = (_one(dd, 1), _one(dd, 2), _one(dd, 3))
        if _one(r, 3) is not None:
            out["hessian_stats"] = (_one(r, 3), _one(r, 4), _one(r, 5))
    cond = _one(f, 3)
    if cond is not None:
        c = pb_decode(cond)
        out["na_value"] = bool(_one(c, 1, 0))
        out["attribute"] = _one(c, 2)
        out["n_cond"] = _one(c, 4)
        out["split_score"] = _one(c, 6, 0.0)
        out["n_pos"] = _one(c, 7)
        cc = pb_decode(_one(c, 3))
        for ff, _, v in cc:
            if ff == 6:
                out["discretized_threshold"] = _one(pb_decode(v), 1)
            elif ff == 5:
                bm = _one(pb_decode(v), 1, b"")
                out["positive_categories"] = [i for i in range(len(bm) * 8) if bm[i // 8] >> (i & 7) & 1]
            elif ff == 4:
                packed, elems, i = _one(pb_decode(v), 1, b""), [], 0
                while i < len(packed):
                    x, sh = 0, 0
                    while True:
                        c8 = packed[i]
                        i += 1
                        x |= (c8 & 0x7F) << sh
                        sh += 7
                        if not c8 & 0x80:
                            break
                    elems.append(x)
                out["positive_categories"] = elems
            elif ff == 2:
                out["higher_threshold"] = _one(pb_decode(v), 1)
    return out


def read_data_spec(path):
    """dataset.proto.DataSpecification (data_spec.pb of any YDF model directory) -> ([column dict], created_num_rows):
    type, name, NumericalSpec.mean, DiscretizedNumericalSpec.boundaries, CategoricalSpec (most_frequent_value,
    number_of_unique_values, vocabulary {key: index})."""
    spec = pb_decode(open(path, "rb").read())
    columns = []
    for f, w, v in spec:
        if f == 1:
            c = pb_decode(v)
            col = {"type": _one(c, 1), "name": _one(c, 2).decode()}
            num = _one(c, 5)
            if num is not None:
                col["mean"] = _one(pb_decode(num), 1, 0.0)
            disc = _one(c, 8)
            if disc is not None:
                col["boundaries"] = np.frombuffer(_one(pb_decode(disc), 1, b""), dtype="<f4")
            cat = _one(c, 6)
            if cat is not None:
                cc = pb_decode(cat)
                col["most_frequent_value"] = _one(cc, 1, 0)
                col["number_of_unique_values"] = _one(cc, 2, 0)
                vocab = {}
                for ff, _, vv in cc:
                    if ff == 7:
                        e = pb_decode(vv)
                        vocab[_one(e, 1).decode()] = _one(pb_decode(_one(e, 2, b"")), 1, 0)
                col["vocabulary"] = vocab
            columns.append(col)
    return columns, _one(spec, 2)


def read_ydf_model(path):
    """Reads header / GBT header / nodes of a YDF GBT model directory (ours or the reference's)."""
    h = pb_decode(open(os.path.join(path, "header.pb"), "rb").read())
    g = pb_decode(open(os.path.join(path, "gradient_boosted_trees_header.pb"), "rb").read())
    nodes = [decode_node(r) for r in read_blob_sequence(os.path.join(path, "nodes-00000-of-00001"))]
    columns, created_num_rows = read_data_spec(os.path.join(path, "data_spec.pb"))
    return {
        "name": _one(h, 1).decode(), "task": _one(h, 2), "label_col_idx": _one(h, 3),
        "input_features": [v for f, _, v in h if f == 5],
        "num_trees": _one(g, 2), "loss": _one(g, 3),
        "initial_predictions": [v for f, _, v in g if f == 4],
        "node_format": _one(g, 7).decode(), "num_trees_per_iter": _one(g, 5, 1),
        "validation_loss": _one(g, 6), "early_stopping_triggered": bool(_one(g, 11, 0)),
        "training_logs": [dict((("number_of_trees", "training_loss", "training_secondary", "validation_loss",
                                 "validation_secondary")[f - 1], v) for f, _, v in pb_decode(e) if 1 <= f <= 5)
                          for ff, _, e in pb_decode(_one(g, 8, b"")) if ff == 1],
        "nodes": nodes, "columns": columns, "created_num_rows": created_num_rows,
    }


# ---- generic evaluation of a YDF GBT model directory (tests) ----------------------------------------
def predict_ydf_model(model: dict, columns: dict) -> np.ndarray:
    """Evaluates a model read by read_ydf_model on raw columns: {name: float array (NaN = missing) for
    NUMERICAL columns, array of str ("" = missing) for CATEGORICAL columns}.  Follows the reference's condition
    evaluation (model/decision_tree/decision_tree.cc:724-812): Higher: value >= threshold; DiscretizedHigher: bin >=
    threshold; Contains{Vector,Bitmap}: dictionary index in the positive set (out-of-dictionary = 0); a missing
    value takes NodeCondition.na_value.  GBT output = initial prediction + sum of the leaves of every tree
    (sigmoid for the binomial loss; one tree per iteration).  Returns the raw score per row."""
    cols = model["columns"]
    n = len(next(iter(columns.values())))
    values, missing = [], []
    for c in cols:
        if c["name"] not in columns:
            values.append(None); missing.append(None)
            continue
        v = columns[c["name"]]
        if c["type"] == 4:  # CATEGORICAL: dictionary index, 0 = out of dictionary
            vocab = c.get("vocabulary", {})
            keys = np.asarray(v, dtype=object)
            idx = np.fromiter((vocab.get(str(k), 0) for k in keys), dtype=np.int64, count=n)
            miss = np.fromiter((k is None or str(k) == "" for k in keys), dtype=bool, count=n)
            values.append(idx); missing.append(miss)
        elif c["type"] == 9:  # DISCRETIZED_NUMERICAL: bin index = upper_bound(boundaries, x)
            x = np.asarray(v, dtype=np.float32)
            values.append(np.searchsorted(c["boundaries"], x, side="right").astype(np.int64)); missing.append(np.isnan(x))
        else:
            x = np.asarray(v, dtype=np.float32)
            values.append(x); missing.append(np.isnan(x))
    nodes = model["nodes"]
    # pre-order layout: the negative subtree follows its parent, then the positive one (decision_tree.cc:609-646)
    neg = np.full(len(nodes), -1, np.int64)
    pos = np.full(len(nodes), -1, np.int64)
    roots = []

    def link(i):
        if "attribute" not in nodes[i]:
            return i + 1
        neg[i] = i + 1
        j = link(i + 1)
        pos[i] = j
        return link(j)

    import sys
    sys.setrecursionlimit(max(10000, sys.getrecursionlimit()))
    i = 0
    while i < len(nodes):
        roots.append(i)
        i = link(i)
    out = np.full(n, model["initial_predictions"][0], dtype=np.float32)
    rows = np.arange(n)
    for r in roots:
        node = np.full(n, r, dtype=np.int64)
        while True:
            active = np.array([("attribute" in nodes[k]) for k in node]) if n < 64 else None
            uniq = np.unique(node)
            moved = False
            for k in uniq:
                nd = nodes[k]
                if "attribute" not in nd:
                    continue
                sel = rows[node == k]
                a = nd["attribute"]
                v, miss = values[a][sel], missing[a][sel]
                if "higher_threshold" in nd:
                    go = v >= np.float32(nd["higher_threshold"])
                elif "discretized_threshold" in nd:
                    go = v >= nd["discretized_threshold"]
                else:
                    go = np.isin(v, np.asarray(nd["positive_categories"], dtype=np.int64))
                go = np.where(miss, bool(nd["na_value"]), go)
                node[sel] = np.where(go, pos[k], neg[k])
                moved = True
            if not moved:
                break
        out += np.array([nodes[k]["top_value"] for k in node], dtype=np.float32)
    return out
