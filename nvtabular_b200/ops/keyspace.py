"""Key spaces: how a user column (ints, floats, strings, list leaves, or a
multi-column combination) becomes the int32/int64 key column the hash kernels
consume, and how keys are decoded back for the parquet artefacts.

All mappings are ORDER-PRESERVING, so the vocabulary tie rule (size desc, key
asc — reference nvtabular/ops/categorify.py:1300,1316) holds on the encoded
keys.  Host work here is O(#distinct strings), never O(#rows); row-level
remaps are device gathers.
"""
from typing import List, Optional, Sequence

import numpy as np
import pandas as pd
import torch

from .. import engine
from ..column import Column

_SIGN_FLIP = 0x7FFFFFFFFFFFFFFF
_I32_MIN = np.iinfo(np.int32).min


def _leaf(col: Column) -> Column:
    from .fill import materialize
    col = materialize(col)
    return Column(col.data, col.validity, None, col.dictionary, None, col.is_bool)


def _float_to_key(col: Column) -> Column:
    """float -> int64 with the same ordering (IEEE total order on finite values);
    NaN becomes null."""
    from ..column import pack_validity, unpack_validity
    x = col.data.to(torch.float64) + 0.0           # -0.0 -> +0.0
    b = x.view(torch.int64)
    key = torch.where(b >= 0, b, b ^ _SIGN_FLIP)
    isnan = torch.isnan(x)
    validity = col.validity
    if bool(isnan.any()):
        valid = unpack_validity(col.validity, x.numel(), x.device) & ~isnan
        validity = pack_validity(valid)
    return Column(key, validity)


def _key_to_float(keys: np.ndarray) -> np.ndarray:
    k = keys.astype(np.int64)
    b = np.where(k >= 0, k, k ^ np.int64(_SIGN_FLIP))
    return b.view(np.float64)


class KeySpace:
    """Single-column key space.  kind: int | float | str."""

    def __init__(self, kind: str, dictionary: Optional[np.ndarray] = None, np_dtype=None):
        self.kind = kind
        self.dictionary = dictionary          # sorted distinct strings (kind == "str")
        self.np_dtype = np_dtype              # original numeric dtype, for decode
        self._lut_cache = {}

    @classmethod
    def for_columns(cls, cols: Sequence[Column], sync: bool = True) -> "KeySpace":
        """Union key space of several columns (joint encoding / partitions).

        Under torch.distributed (one process per GPU) the key space must be IDENTICAL on
        every rank before keys are exchanged by owner: string dictionaries are rank-local,
        so with `sync` the ranks all-gather their distinct strings and build the same union
        dictionary (and agree on the numeric width; a rank with no rows adopts the others').
        This is a collective: every rank must make the same sequence of synced calls.
        `sync=False` is for callers that have already agreed on a numeric dtype."""
        kind, np_dtype, uni = None, None, None
        if cols:
            first = cols[0]
            if first.is_string:
                if not all(c.is_string for c in cols):
                    raise TypeError("cannot jointly encode string and non-string columns")
                parts = [c.dictionary for c in cols if len(c.dictionary)]
                uni = np.array(sorted(set(np.concatenate(parts).tolist())), dtype=object) if parts \
                    else np.array([], dtype=object)
                kind = "str"
            elif first.data.dtype in (torch.float32, torch.float64):
                kind, np_dtype = "float", first.np_dtype
            else:
                kind = "int"
                np_dtype = np.dtype("int64") if any(c.data.dtype == torch.int64 for c in cols) else np.dtype("int32")
        if sync:
            from ..dist import all_gather_object, world
            if world()[0] > 1:
                seen = all_gather_object((kind, str(np_dtype) if np_dtype is not None else None,
                                          uni.tolist() if uni is not None else None))
                kinds = {k for k, _, _ in seen if k is not None}
                if len(kinds) > 1:
                    raise TypeError(f"ranks disagree on the key type of a column group: {sorted(kinds)}")
                kind = kinds.pop() if kinds else None
                if kind == "str":
                    uni = np.array(sorted(set(x for _, _, d in seen if d for x in d)), dtype=object)
                elif kind == "int":
                    np_dtype = np.dtype("int64") if any(d == "int64" for _, d, _ in seen) else np.dtype("int32")
                elif kind == "float":
                    np_dtype = np.dtype("float64") if any(d == "float64" for _, d, _ in seen) else np.dtype("float32")
        if kind is None:                       # no rows anywhere
            return cls("int", None, np.dtype("int64"))
        return cls(kind, uni, np_dtype)

    def extend(self, cols: Sequence[Column]) -> "KeySpace":
        if self.kind != "str":
            return self
        return KeySpace.for_columns([Column(torch.zeros(0, dtype=torch.int32), dictionary=self.dictionary)] + list(cols))

    # -- data column -> key column -------------------------------------------------
    def keys_for(self, col: Column) -> Column:
        col = _leaf(col)
        if self.kind == "int":
            if col.is_string or col.data.dtype in (torch.float32, torch.float64):
                if col.data.dtype in (torch.float32, torch.float64) and not col.is_string:
                    # a float column against an integer vocabulary (e.g. pandas turned an int
                    # column with nulls into float64): integral values keep their identity
                    x = col.data.to(torch.float64)
                    from ..column import pack_validity, unpack_validity
                    bad = torch.isnan(x) | (x != torch.trunc(x))
                    validity = col.validity
                    data = torch.where(bad, torch.zeros_like(x), x).to(torch.int64)
                    if bool(bad.any()):
                        # NaN -> null; a fractional value can never be in an int vocabulary:
                        # give it a key no integer column produces twice (still OOV)
                        valid = unpack_validity(col.validity, x.numel(), x.device) & ~torch.isnan(x)
                        validity = pack_validity(valid)
                    return Column(data, validity)
                raise TypeError("string column against an integer vocabulary")
            if col.data.dtype == torch.uint8:
                return Column(col.data.to(torch.int32), col.validity)
            return Column(col.data, col.validity)
        if self.kind == "float":
            return _float_to_key(col)
        # strings: partition-local codes -> global order-preserving ids (device gather)
        if not col.is_string:
            raise TypeError("non-string column against a string vocabulary")
        lut = self._string_lut(col.dictionary, col.data.device)
        if lut is None:
            return Column(col.data, col.validity)
        idx = col.data.to(torch.int64)
        if lut.numel() == 0:
            return Column(torch.full_like(idx, -1), col.validity)
        return Column(lut[idx.clamp(0, lut.numel() - 1)], col.validity)

    def _string_lut(self, part_dict: np.ndarray, device):
        if len(part_dict) == len(self.dictionary) and (len(part_dict) == 0 or
                                                        np.array_equal(part_dict, self.dictionary)):
            return None                                   # identical dictionary: codes are ids
        key = (id(part_dict), len(part_dict))
        hit = self._lut_cache.get(key)
        if hit is not None and hit[0] is part_dict:
            return hit[1]
        if len(self.dictionary):
            pos = np.searchsorted(self.dictionary.astype(str), part_dict.astype(str))
            pos_c = np.clip(pos, 0, len(self.dictionary) - 1)
            found = self.dictionary[pos_c] == part_dict
            ids = np.where(found, pos_c, -1 - np.arange(len(part_dict)))   # unseen -> distinct negatives
        else:
            ids = -1 - np.arange(len(part_dict))
        lut = torch.from_numpy(ids.astype(np.int64)).to(device)
        self._lut_cache = {key: (part_dict, lut)}
        return lut

    # -- keys -> original values (host, O(U)) ---------------------------------------
    def decode(self, keys: np.ndarray) -> np.ndarray:
        if self.kind == "int":
            return keys.astype(self.np_dtype or np.int64)
        if self.kind == "float":
            return _key_to_float(keys).astype(self.np_dtype or np.float64)
        out = np.empty(len(keys), dtype=object)
        ok = (keys >= 0) & (keys < len(self.dictionary))
        out[ok] = self.dictionary[keys[ok]]
        out[~ok] = None
        return out

    def encode_values(self, values) -> np.ndarray:
        """host values (a vocabulary read from parquet / passed by the user) -> keys."""
        ser = pd.Series(values)
        if self.kind == "str":
            idx = pd.Index(self.dictionary)
            return idx.get_indexer(ser.astype(object)).astype(np.int64)
        if self.kind == "float":
            x = ser.to_numpy(dtype=np.float64) + 0.0
            b = x.view(np.int64)
            return np.where(b >= 0, b, b ^ np.int64(_SIGN_FLIP))
        return ser.to_numpy(dtype=np.int64)

    def hash_column(self, col: Column) -> Optional[Column]:
        """column whose VALUE hash drives OOV buckets (None = hash the key itself)."""
        col = _leaf(col)
        if self.kind == "str":
            from .hash_bucket import string_hash_column
            return string_hash_column(col)
        if self.kind == "float":
            return Column(col.data, col.validity)
        return None


class ComboKeySpace:
    """Multi-column combination key (encode_type="combo", JoinGroupby groups).

    Fast path: two int32 columns are packed directly, (a << 32) | (b ^ 2^31).
    General path: every component is first replaced by its dense,
    order-preserving rank (null = rank 0) and the ranks are packed pairwise; a
    third and later component re-ranks the running pair first."""

    def __init__(self, spaces: List[KeySpace], rank_vocabs=None, rank_keys=None):
        self.spaces = spaces
        self.rank_vocabs = rank_vocabs      # per stage: engine.Vocab of sorted keys, or None (direct)
        self.rank_keys = rank_keys          # per stage: host sorted key arrays (decode)

    @property
    def direct(self) -> bool:
        return self.rank_vocabs is None

    @staticmethod
    def can_pack_direct(cols: Sequence[Column]) -> bool:
        return len(cols) == 2 and all((not c.is_string) and c.data.dtype == torch.int32 for c in cols)

    @classmethod
    def fit(cls, partitions: Sequence[Sequence[Column]], ncomp: Optional[int] = None,
            sync: bool = True) -> "ComboKeySpace":
        """partitions: per partition, the component columns (leaves).  `ncomp` must be given
        when a rank may hold no partition (every rank runs the same collectives).  `sync=False`
        builds a rank-local space and runs no collective (a table every rank holds whole)."""
        ncomp = ncomp if ncomp is not None else len(partitions[0])
        spaces = [KeySpace.for_columns([p[j] for p in partitions], sync=sync) for j in range(ncomp)]
        # decided from the (rank-synchronised) spaces, so every rank takes the same path
        if ncomp == 2 and all(s.kind == "int" and s.np_dtype == np.dtype("int32") for s in spaces) and \
                all(cls.can_pack_direct(p) for p in partitions):
            return cls(spaces)
        self = cls(spaces, [], [])
        # stage j ranks component j; stage ncomp+k ranks the k-th running pair
        running = None
        for j in range(ncomp):
            comp_keys = [spaces[j].keys_for(p[j]) for p in partitions]
            vocab, host = cls._rank_vocab(comp_keys, sync)
            self.rank_vocabs.append(vocab)
            self.rank_keys.append(host)
            ranks = [cls._rank(vocab, k) for k in comp_keys]
            if running is None:
                running = ranks
            else:
                packed = [engine.pack_keys2(a, b) for a, b in zip(running, ranks)]
                if j < ncomp - 1:
                    pv, ph = cls._rank_vocab(packed, sync)
                    self.rank_vocabs.append(pv)
                    self.rank_keys.append(ph)
                    running = [cls._rank(pv, k) for k in packed]
        return self

    @staticmethod
    def _rank_vocab(key_cols: Sequence[Column], sync: bool = True):
        from ..dist import global_merge
        agg = engine.HashAgg(0)
        for k in key_cols:
            agg.insert(k)
        # identical on every rank (single GPU, or sync=False: an export)
        keys, _, _, _, _ = global_merge(agg) if sync else agg.export()
        keys, _ = torch.sort(keys)
        return engine.Vocab.from_arrays(keys), keys.cpu().numpy()

    @staticmethod
    def _rank(vocab, key: Column) -> Column:
        # null -> rank 0 (kept valid so "some nulls" tuples stay ordinary keys),
        # unseen -> INT32_MIN + 1 (never a rank), seen -> 1 + position
        r = vocab.encode(key, null_label=0, oov_label=_I32_MIN + 1, first_label=1, out_dtype=np.int32)
        return Column(r, key.validity)

    def keys_for(self, cols: Sequence[Column]) -> Column:
        cols = [_leaf(c) for c in cols]
        if self.direct:
            ks = [s.keys_for(c) for s, c in zip(self.spaces, cols)]
            return engine.pack_keys2(ks[0], ks[1])
        stage = 0
        running = None
        n = len(cols)
        for j in range(n):
            k = self.spaces[j].keys_for(cols[j])
            r = self._rank(self.rank_vocabs[stage], k)
            stage += 1
            if running is None:
                running = r
            else:
                packed = engine.pack_keys2(running, r)
                if j < n - 1:
                    running = self._rank(self.rank_vocabs[stage], packed)
                    stage += 1
                else:
                    running = packed
        return running

    def decode(self, keys: np.ndarray) -> List[np.ndarray]:
        """packed keys -> one host array per component (None where null)."""
        n = len(self.spaces)
        if self.direct:
            a, b = engine.unpack_keys2(keys)
            outs = []
            for s, v in zip(self.spaces, (a, b)):
                vals = s.decode(v.astype(np.int64)).astype(object)
                vals[v == _I32_MIN] = None
                outs.append(vals)
            return outs
        comps = [None] * n
        cur = keys
        # rank stages were appended as: c0, c1, [pair], c2, [pair], ...
        stage_of_comp, stage_of_pair, s = {}, {}, 0
        for j in range(n):
            stage_of_comp[j] = s
            s += 1
            if 0 < j < n - 1:
                stage_of_pair[j] = s
                s += 1
        for j in range(n - 1, 0, -1):
            a, b = engine.unpack_keys2(cur)
            comps[j] = self._unrank(stage_of_comp[j], b, self.spaces[j])
            if j - 1 >= 1:
                pk = self.rank_keys[stage_of_pair[j - 1]]
                cur = pk[np.clip(a.astype(np.int64) - 1, 0, len(pk) - 1)]
            else:
                comps[0] = self._unrank(stage_of_comp[0], a, self.spaces[0])
        return comps

    def _unrank(self, stage, ranks, space):
        host = self.rank_keys[stage]
        r = ranks.astype(np.int64)
        vals = space.decode(host[np.clip(r - 1, 0, max(len(host) - 1, 0))]) if len(host) else \
            np.empty(len(r), dtype=object)
        vals = vals.astype(object)
        vals[(r <= 0)] = None
        return vals

    def first_component_null_t(self, keys: torch.Tensor) -> torch.Tensor:
        """device version of first_component_null for packed two-component keys (no host round trip
        over tens of millions of group keys); falls back to the host path for deeper combinations"""
        if len(self.spaces) == 2 or self.direct:
            a = keys >> 32                                        # arithmetic: the first component, sign-extended
            return (a == int(_I32_MIN)) if self.direct else (a <= 0)
        return torch.from_numpy(self.first_component_null(keys.cpu().numpy())).to(keys.device)

    def first_component_null(self, keys: np.ndarray) -> np.ndarray:
        a, _ = engine.unpack_keys2(keys) if len(self.spaces) == 2 or self.direct else (None, None)
        if a is None:
            comps = self.decode(keys)
            return np.array([v is None for v in comps[0]], dtype=bool)
        return (a == _I32_MIN) if self.direct else (a <= 0)
