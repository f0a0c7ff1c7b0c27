"""Host side of `solver` (J/Solver.java:161-432): point matches from stitching results or interest-point
correspondences, the view -> tile grouping, fixed tiles, pre-alignment, the tile colouring of the device relaxation
(bs_solve_tiles), the ONE_ROUND_ITERATIVE link removal and the registrations written back to the XML.

Coordinates: every point is a world position under the views' current registrations, and a tile's model maps those
world positions to the new ones, so a view's new registration is the tile model applied after its current one.  A link
(a, b), a < b, holds the matches p (tile a) <-> q (tile b); a tile t fits M_t(own point) ~ M_u(partner point)."""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from . import matching as bm
from .spimdata import SpimData2

METHODS = ("ONE_ROUND_SIMPLE", "ONE_ROUND_ITERATIVE", "TWO_ROUND_SIMPLE", "TWO_ROUND_ITERATIVE")
_MODEL_NAMES = {"TRANSLATION": "TranslationModel3D", "RIGID": "RigidModel3D", "AFFINE": "AffineModel3D"}


@dataclass
class Problem:
    """One solve: tiles 0..T-1, links (L, 2) with a < b in ascending (a, b) order, and the matches of link l in
    rows match_offsets[l]:match_offsets[l + 1] of p / q / w."""
    n_tiles: int
    links: np.ndarray
    match_offsets: np.ndarray
    p: np.ndarray
    q: np.ndarray
    w: np.ndarray
    fixed: np.ndarray = field(default=None)


def model_name(transformation, regularization):
    """Name of the written <ViewTransform>: the simple class name of the model createModelInstance builds (recalled,
    PARITY_GAPS S4)."""
    base = _MODEL_NAMES[transformation.upper()]
    return base if regularization.upper() == "NONE" else "Interpolated" + base


# ------------------------------------------------------------------------------------------------ grouping, matches
def tile_keys(data: SpimData2, views, group_tiles=False, group_illums=False, group_channels=False, split_timepoints=False):
    """{view: key}; views with the same key share one tile.  --splitTimepoints puts all views of a timepoint in one tile;
    otherwise every --group* flag drops that attribute from the key; with no flag every view is its own tile."""
    keys = {}
    for v in views:
        a = data.setups[v[1]].attributes
        if split_timepoints:
            keys[v] = (v[0],)
        elif not (group_tiles or group_illums or group_channels):
            keys[v] = (v[0], v[1])
        else:
            keys[v] = (v[0], a.get("angle", 0), None if group_channels else a.get("channel", 0),
                       None if group_illums else a.get("illumination", 0), None if group_tiles else a.get("tile", v[1]))
    return keys


def stitching_matches(data: SpimData2, tile_of, views):
    """Matches of the stored stitching results (J/Solver.java:398-432): results whose hash differs from the hash of the
    first views' current registrations are stale and dropped; every other result (A, B, R, r, overlap box) gives the 8
    corners c of the box as matches A: c <-> B: R^-1(c) of weight r.  Returns (ta, tb, p, q, w, n_stale)."""
    sel = set(views)
    ta, tb, ps, qs, ws = [], [], [], [], []
    stale = 0
    for res in data.stitching_results():
        ga = res["pair"][0] if isinstance(res["pair"][0][0], tuple) else (res["pair"][0],)
        gb = res["pair"][1] if isinstance(res["pair"][1][0], tuple) else (res["pair"][1],)
        if SpimData2.transform_hash(data.registrations[ga[0]], data.registrations[gb[0]]) != res["hash"]:
            stale += 1
            continue
        va, vb = [v for v in ga if v in sel], [v for v in gb if v in sel]
        if not va or not vb or tile_of[va[0]] == tile_of[vb[0]] or len(res["bbox"]) != 6:
            continue
        lo, hi = res["bbox"][:3], res["bbox"][3:]
        c = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
        R = np.vstack([np.asarray(res["shift"], dtype=np.float64).reshape(3, 4), [0, 0, 0, 1]])
        Ri = np.linalg.inv(R)[:3]
        ta.append(np.full(8, tile_of[va[0]]))
        tb.append(np.full(8, tile_of[vb[0]]))
        ps.append(c)
        qs.append(c @ Ri[:, :3].T + Ri[:, 3])
        ws.append(np.full(8, float(res["r"])))
    return _cat(ta, tb, ps, qs, ws) + (stale,)


def ip_matches(ips, tile_of, views, labels, label_weights):
    """Matches of the stored correspondences: every correspondence between two selected views whose labels are both
    in ``labels``, once per pair (from the side that sorts first), with both points at their world positions and the
    weight of the first point's label.  ``ips``: commands._InterestPoints read with correspondence tables."""
    sel = set(views)
    weight = dict(zip(labels, label_weights))
    ta, tb, ps, qs, ws = [], [], [], [], []
    for (v, lab) in sorted(ips.table):
        rows, keys = ips.table[(v, lab)]
        if len(rows) == 0:
            continue
        ids = ips.ids[(v, lab)]
        order = np.argsort(ids, kind="stable")
        for k, (pv, pl) in sorted(keys.items()):
            if pv not in sel or pl not in weight or (pv, pl) not in ips.world or (pv, pl) <= (v, lab):
                continue
            if tile_of[pv] == tile_of[v]:
                continue
            r = rows[rows[:, 2] == k]
            pids = ips.ids[(pv, pl)]
            porder = np.argsort(pids, kind="stable")
            ia = order[np.searchsorted(ids, r[:, 0].astype(np.int64), sorter=order)]
            ib = porder[np.searchsorted(pids, r[:, 1].astype(np.int64), sorter=porder)]
            ta.append(np.full(len(r), tile_of[v]))
            tb.append(np.full(len(r), tile_of[pv]))
            ps.append(ips.world[(v, lab)][ia])
            qs.append(ips.world[(pv, pl)][ib])
            ws.append(np.full(len(r), float(weight[lab])))
    return _cat(ta, tb, ps, qs, ws)


def _cat(ta, tb, ps, qs, ws):
    if not ta:
        return (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0))
    return (np.concatenate(ta).astype(np.int64), np.concatenate(tb).astype(np.int64), np.concatenate(ps).astype(np.float64),
            np.concatenate(qs).astype(np.float64), np.concatenate(ws).astype(np.float64))


def build_problem(n_tiles, ta, tb, p, q, w) -> Problem:
    """Orient every match so that its link is (a, b) with a < b and sort the matches by link (stable)."""
    swap = ta > tb
    a, b = np.where(swap, tb, ta), np.where(swap, ta, tb)
    p, q = np.where(swap[:, None], q, p), np.where(swap[:, None], p, q)
    order = np.lexsort((b, a))
    a, b, p, q, w = a[order], b[order], p[order], q[order], w[order]
    links, start = np.unique(np.stack([a, b], axis=1), axis=0, return_index=True)
    offsets = np.append(np.sort(start), len(a)).astype(np.int64)
    return Problem(int(n_tiles), links.reshape(-1, 2).astype(np.int64), offsets, np.ascontiguousarray(p),
                   np.ascontiguousarray(q), np.ascontiguousarray(w))


def drop_link(prob: Problem, l) -> Problem:
    keep = np.ones(len(prob.w), dtype=bool)
    keep[prob.match_offsets[l]:prob.match_offsets[l + 1]] = False
    n = np.diff(prob.match_offsets)
    n = np.delete(n, l)
    return Problem(prob.n_tiles, np.delete(prob.links, l, axis=0), np.concatenate([[0], np.cumsum(n)]).astype(np.int64),
                   prob.p[keep], prob.q[keep], prob.w[keep], prob.fixed)


def neighbours(n_tiles, links):
    nb = [[] for _ in range(n_tiles)]
    for l, (a, b) in enumerate(np.asarray(links).tolist()):
        nb[a].append((b, l))
        nb[b].append((a, l))
    return nb


def colouring(n_tiles, links):
    """Greedy colouring in tile-index order: each tile takes the smallest colour none of its lower-index neighbours
    has.  Returns (colour per tile, colour offsets (C + 1,), tiles ordered by colour then index)."""
    nb = neighbours(n_tiles, links)
    col = np.zeros(n_tiles, dtype=np.int64)
    for t in range(n_tiles):
        used = {int(col[u]) for u, _ in nb[t] if u < t}
        c = 0
        while c in used:
            c += 1
        col[t] = c
    order = np.lexsort((np.arange(n_tiles), col)).astype(np.int32)
    ncol = int(col.max()) + 1 if n_tiles else 0
    offsets = np.searchsorted(col[order], np.arange(ncol + 1)).astype(np.int32)
    return col, offsets, order


# ------------------------------------------------------------------------------------------------ solve
def tile_matches(prob: Problem, t, partners=None):
    """(own points, partner tile per match, partner points, weights) of tile t, optionally only with ``partners``."""
    xs, us, zs, ws = [], [], [], []
    for l, (a, b) in enumerate(prob.links.tolist()):
        if t not in (a, b):
            continue
        u = b if a == t else a
        if partners is not None and u not in partners:
            continue
        s = slice(prob.match_offsets[l], prob.match_offsets[l + 1])
        xs.append(prob.p[s] if a == t else prob.q[s])
        zs.append(prob.q[s] if a == t else prob.p[s])
        us.append(np.full(s.stop - s.start, u))
        ws.append(prob.w[s])
    if not xs:
        return np.zeros((0, 3)), np.zeros(0, np.int64), np.zeros((0, 3)), np.zeros(0)
    return np.concatenate(xs), np.concatenate(us), np.concatenate(zs), np.concatenate(ws)


def apply_models(M, u, z):
    """M[u[i]] applied to z[i]."""
    return np.einsum("nij,nj->ni", M[u][:, :, :3], z) + M[u][:, :, 3]


def prealign(prob: Problem, model: bm.Model):
    """TileConfiguration.preAlign: breadth first from the fixed tiles (tile 0 when none is fixed); each unaligned
    neighbour of the current tile is fitted to its matches with the tiles aligned so far and becomes aligned.  A fit
    that fails leaves the identity.  Tiles no fixed tile reaches keep the identity."""
    M = np.tile(np.eye(3, 4), (prob.n_tiles, 1, 1))
    nb = neighbours(prob.n_tiles, prob.links)
    seeds = [int(t) for t in np.nonzero(prob.fixed)[0]] or ([0] if prob.n_tiles else [])
    aligned = set(seeds)
    queue = list(seeds)
    while queue:
        r = queue.pop(0)
        for u, _ in sorted(nb[r]):
            if u in aligned:
                continue
            x, pu, z, w = tile_matches(prob, u, aligned)
            if len(x) >= max(model.min_matches, 1):
                F, ok = model.fit(x[None], apply_models(M, pu, z)[None], w[None])
                if ok[0]:
                    M[u] = F[0]
            aligned.add(u)
            queue.append(u)
    return M


def proceed(errors, max_error, max_plateau_width):
    """The stopping rule after iteration i = len(errors) (errors[k] = E_{k+1}): always go on while i <= the plateau
    width; then go on while E_i > max_error or any |E_i - E_{i-d}| / d > 1e-4 for d = width, width / 2, ... >= 1."""
    i = len(errors)
    if i <= max_plateau_width:
        return True
    go = errors[-1] > max_error
    d = max_plateau_width
    while d >= 1:
        go |= abs((errors[-1] - errors[-1 - d]) / d) > 1e-4
        d //= 2
    return bool(go)


def not_converged(tile_error, relative_threshold, absolute_threshold):
    """SimpleIterativeConvergenceStrategy: (avg * rel < max and max > 0.95) or avg > abs over the tile errors."""
    avg, mx = float(np.mean(tile_error)), float(np.max(tile_error))
    return (avg * relative_threshold < mx and mx > 0.95) or avg > absolute_threshold


def worst_link(prob: Problem, link_max):
    """MaxErrorLinkRemoval: the link holding the largest point-match distance among links whose two tiles both keep
    another link (no tile is cut off); the first such link on ties.  None when no link qualifies."""
    deg = np.bincount(prob.links.ravel(), minlength=prob.n_tiles)
    ok = (deg[prob.links[:, 0]] > 1) & (deg[prob.links[:, 1]] > 1)
    if not ok.any():
        return None
    return int(np.argmax(np.where(ok, link_max, -np.inf)))


def solve(ctx, prob: Problem, model: bm.Model, method="ONE_ROUND_SIMPLE", max_error=5.0, max_iterations=10000,
          max_plateau_width=200, relative_threshold=3.5, absolute_threshold=7.0):
    """Pre-align and relax one problem on the device; ONE_ROUND_ITERATIVE repeats with max_error = inf, dropping the
    worst link after each round that has not converged.  Returns (models (T, 3, 4), removed links as (a, b) tile
    pairs, stats)."""
    iterative = method == "ONE_ROUND_ITERATIVE"
    removed, rounds = [], 0
    kw = dict(transformation=model.tm, regularization=model.rm, lam=model.lam,
              max_error=float("inf") if iterative else float(max_error), max_iterations=int(max_iterations),
              max_plateau_width=int(max_plateau_width))
    while True:
        rounds += 1
        _, coff, corder = colouring(prob.n_tiles, prob.links)
        M0 = prealign(prob, model)
        M, st, tile_err, _, link_max = ctx.solve_tiles(coff, corder, prob.fixed, prob.links, prob.match_offsets, prob.p,
                                                        prob.q, prob.w, M0, **kw)
        if not iterative or not not_converged(tile_err, relative_threshold, absolute_threshold):
            break
        l = worst_link(prob, link_max)
        if l is None:
            break
        removed.append(tuple(int(v) for v in prob.links[l]))
        prob = drop_link(prob, l)
    st = dict(st, rounds=rounds, tile_error=tile_err)
    return M, removed, st


# ------------------------------------------------------------------------------------------------ the command
def run(xml_path, ctx, source, labels=None, label_weights=None, method="ONE_ROUND_SIMPLE", transformation_model="AFFINE",
        regularization_model="RIGID", regularization_lambda=0.1, max_error=5.0, max_iterations=10000,
        max_plateau_width=200, relative_threshold=3.5, absolute_threshold=7.0, fixed_views=None,
        disable_fixed_views=False, group_tiles=None, group_illums=None, group_channels=None, split_timepoints=None,
        registration_tp="TIMEPOINTS_INDIVIDUALLY", view_selection=None, dry_run=False):
    from . import n5 as bn5
    from .commands import _InterestPoints
    m = method.upper()
    if m not in METHODS:
        raise ValueError(f"--method {method}")
    if m.startswith("TWO_ROUND"):
        raise NotImplementedError(f"solver --method {m} is not implemented")
    if registration_tp.upper() != "TIMEPOINTS_INDIVIDUALLY":
        raise NotImplementedError(f"solver -rtp {registration_tp} is not implemented")
    src = source.upper()
    if src not in ("STITCHING", "IP"):
        raise ValueError(f"-s {source}")
    model = bm.Model(transformation_model, regularization_model, regularization_lambda)
    data = SpimData2.load(xml_path)
    views = sorted(data.select_views(**view_selection) if view_selection else data.view_ids())
    if src == "IP":
        labels = list(labels or [])
        if not labels:
            raise ValueError("No labels specified.")
        label_weights = [1.0] * len(labels) if not label_weights else [float(x) for x in label_weights]
        if len(label_weights) != len(labels):
            raise ValueError("You need to specify as many weights as labels, or do not specify weights at all")
        dflt = False
    else:
        dflt = True                                     # stitching groups a tile's channels and illuminations
    keys = tile_keys(data, views, bool(group_tiles), dflt if group_illums is None else bool(group_illums),
                     dflt if group_channels is None else bool(group_channels), bool(split_timepoints))
    key_order = list(dict.fromkeys(keys[v] for v in views))
    cand = {v: key_order.index(keys[v]) for v in views}

    stale = 0
    if src == "STITCHING":
        ta, tb, p, q, w, stale = stitching_matches(data, cand, views)
    else:
        base = os.path.join(os.path.dirname(os.path.abspath(xml_path)), data.root.findtext("BasePath") or ".")
        regs = {v: data.model(*v) for v in views}
        ips = _InterestPoints(bn5.N5Store(os.path.join(base, "interestpoints.n5")), views, labels, regs, tables=True)
        ta, tb, p, q, w = ip_matches(ips, cand, views, labels, label_weights)

    # tiles of the solve: the candidate tiles with at least one link, in candidate order
    used = np.unique(np.concatenate([ta, tb])) if len(ta) else np.zeros(0, np.int64)
    remap = np.full(len(key_order), -1, np.int64)
    remap[used] = np.arange(len(used))
    tile_of = {v: int(remap[cand[v]]) for v in views if remap[cand[v]] >= 0}
    unconnected = [v for v in views if v not in tile_of]
    stats = dict(stale_results=stale, unconnected_views=unconnected, iterations=0, rounds=0, skipped_fits=0)
    if len(used) == 0:
        return dict(models={}, removed=[], stats=stats)
    prob = build_problem(len(used), remap[ta], remap[tb], p, q, w)

    if disable_fixed_views:
        fixed_v = set()
    elif fixed_views:
        fixed_v = {tuple(int(x) for x in (f.split(",") if isinstance(f, str) else f)) for f in fixed_views}
    else:
        fixed_v = {min(v for v in views if v[0] == tp) for tp in sorted({v[0] for v in views})}
    prob.fixed = np.zeros(prob.n_tiles, dtype=np.int32)
    for v in fixed_v:
        if v in tile_of:
            prob.fixed[tile_of[v]] = 1

    M, removed, st = solve(ctx, prob, model, m, max_error, max_iterations, max_plateau_width, relative_threshold,
                           absolute_threshold)
    stats.update(st)
    groups = {}
    for v, t in tile_of.items():
        groups.setdefault(t, []).append(v)
    models = {v: M[t].copy() for v, t in sorted(tile_of.items())}
    name = model_name(model.tm, model.rm)
    for v, Mv in models.items():
        data.add_registration(v, name, Mv)
    if not dry_run:
        data.save(xml_path)
    return dict(models=models, removed=[(sorted(groups[a]), sorted(groups[b])) for a, b in removed], stats=stats)
