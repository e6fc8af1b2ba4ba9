"""The paired comparison per record group (csrc/apo_cand.cu k_cand_group_pairs / k_cand_group_pairs_report): label planes
and tensors that reach its edges, and the exact integer model it is checked against.

For candidate c with reference r = refs[c] and label g < G, the fields are pair_fixtures.pair_model's restricted to the
record positions t with labels[t] == g: a position of another label counts on neither side.  So, summed over g, every
integer field is pair_model's, and G = 1 is pair_model itself.

Label planes (labels(kind, T, G)):
- lanes: t % 64 at G = 64, every lane of a group of 32 its own label;
- mod5: t % 5 at G = 5, peer masks shared by several lanes;
- runs: G contiguous runs (the common held-out split);
- ends: only labels 0 and G - 1;
- tail: label 1 only on the row's last k evaluations (the T mod 1024 tails of pair_fixtures.TAILS), label 0 elsewhere.
Tensors: pair_fixtures' (extreme rows under one label and under alternating labels, one-unit, nulls, RN edges, counts,
shapes with self-pairs, mirrors and PAIR_NONE).

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import numpy as np

import pair_fixtures as pf
import spread_fixtures as sf
from extremes_fixtures import final_rewards, record_final_rewards

NONE = pf.NONE
KINDS = ("lanes", "mod5", "runs", "ends", "tail")
INT_FIELDS = ("n", "wins", "losses", "ties", "candOnly", "refOnly", "D1", "D2")


def labels(kind: str, T: int, G: int = 0, k: int = 1) -> tuple[np.ndarray, int]:
    """(uint8 labels [T], G) of one plane"""
    t = np.arange(T, dtype=np.int64)
    if kind == "lanes":
        return (t % 64).astype(np.uint8), 64
    if kind == "mod5":
        return (t % 5).astype(np.uint8), 5
    if kind == "runs":
        G = G or 8
        return (t * G // T).astype(np.uint8), G
    if kind == "ends":
        G = G or 64
        return np.where(t % 3 == 0, G - 1, 0).astype(np.uint8), G
    if kind == "tail":
        return (t >= T - k).astype(np.uint8), 2
    raise ValueError(kind)


def group_pair_model(fr, ok, refs, lab, G: int) -> list[list[dict]]:
    """[C][G] pairs of rows fr / ok [C][T] under refs [C] and labels [T]"""
    fr, ok = np.atleast_2d(fr), np.atleast_2d(ok).astype(bool)
    lab = np.asarray(lab)[: fr.shape[1]]
    per_g = [pf.pair_model(fr, ok & (lab == g)[None, :], refs) for g in range(G)]
    return [[per_g[g][c] for g in range(G)] for c in range(fr.shape[0])]


def model(dims: np.ndarray, refs, lab, G: int, w=None, recip: bool = False):
    return group_pair_model(*final_rewards(dims, w, recip), refs, lab, G)


def rec_model(recs: np.ndarray, refs, lab, G: int, w=None, recip: bool = False):
    return group_pair_model(*record_final_rewards(recs, w, recip), refs, lab, G)


def summed(per_c: list[dict]) -> dict:
    """the integer fields of one candidate's groups, summed over g"""
    return {f: sum(int(m[f]) for m in per_c) for f in INT_FIELDS}


def all_fixtures():
    """(name, dims, refs, w, labels, G): pair_fixtures' tensors under every label plane, the extreme rows under one label and
    under alternating labels, and a label that holds only each nulls tensor's last evaluations"""
    out = []
    for name, dims, refs, w in pf.all_fixtures():
        T = dims.shape[1]
        if name.startswith("nulls"):
            for k in (1, T % 1024 or 1):
                lab, G = labels("tail", T, k=k)
                out.append((f"{name}_tail{k}", dims, refs, w, lab, G))
            continue
        for kind in KINDS[:4]:
            lab, G = labels(kind, T)
            out.append((f"{name}_{kind}", dims, refs, w, lab, G))
    ex = pf.extreme(8192 + 5)
    out.append(("extreme_one", ex, np.array([1, 0], np.uint32), sf.w_one(), np.zeros(ex.shape[1], np.uint8), 1))
    out.append(("extreme_alt", ex, np.array([1, 0], np.uint32), sf.w_one(), (np.arange(ex.shape[1]) % 2).astype(np.uint8), 2))
    return out


def invariants(gp, pairs, G: int):
    """the per-group pairs of one call [C][G] against its pairs [C]: summed over g every integer field, ref in every group
    (asserts)"""
    for c, p in enumerate(pairs):
        row = gp[c]
        assert all(int(row[g].ref) == int(p.ref) for g in range(G)), c
        for f in ("n", "wins", "losses", "ties", "candOnly", "refOnly"):
            assert sum(int(getattr(row[g], f)) for g in range(G)) == int(getattr(p, f)), (c, f)
        assert sum(row[g].sum for g in range(G)) == p.sum and sum(row[g].sum_sq for g in range(G)) == p.sum_sq, c
