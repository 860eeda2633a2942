"""Static tables of the traffic-junction task, built once on the host.

Reproduces the tables the reference derives in
``ic3net_envs/traffic_junction_env.py:_set_grid`` (:300-319), ``_set_paths_easy``
(:395-410), ``_set_paths`` (:509-523) and ``ic3net_envs/traffic_helper.py``
(``get_road_blocks`` :5-22, ``get_add_mat`` :29-103, ``get_routes`` :156-209), but
with a direct construction instead of the reference's neighbour-search walker:

* roads are two-lane strips, traffic keeps to its lane (right-hand traffic), so a
  car is fully described by a cell and a heading;
* at the k-th junction it meets (k = 1, 2) it applies turn_k: 0 = straight on,
  1 = right turn at the first junction cell, 2 = left turn after the second
  junction cell; later junctions are crossed straight;
* routes are enumerated in the reference's order: arrival point, then turn_1, then
  turn_2, and a first turn that already leads out of the map yields one route.

``tests/test_traffic_tables.py`` checks these tables cell by cell against the
reference's own output (golden fixtures tests/golden/tj_tables_*.npz).
"""
import math

import numpy as np

# headings: (drow, dcol)
DOWN, UP, RIGHT, LEFT = (1, 0), (-1, 0), (0, 1), (0, -1)


def _right_of(hd):     # clockwise turn as seen by the driver
    return {DOWN: LEFT, LEFT: UP, UP: RIGHT, RIGHT: DOWN}[hd]


def _left_of(hd):
    return {DOWN: RIGHT, RIGHT: UP, UP: LEFT, LEFT: DOWN}[hd]


def constants(difficulty, dim):
    """(dims, BASE, OUTSIDE, CAR, vocab, npath): traffic_junction_env.py:103-133."""
    dims = (dim + 1, dim + 1) if difficulty == "easy" else (dim, dim)
    nroad = {"easy": 2, "medium": 4, "hard": 8}[difficulty]
    base = {"easy": 1, "medium": 2, "hard": 4}[difficulty] * (2 * dim)
    npath = math.factorial(nroad) // math.factorial(nroad - 2)
    return dims, base, base, base + 2, base + 3, npath


def road_blocks(h, w, difficulty):
    """Index slices of the road strips, in the reference's numbering order."""
    if difficulty == "easy":
        return [np.s_[h // 2, :], np.s_[:, w // 2]]
    if difficulty == "medium":
        return [np.s_[h // 2 - 1:h // 2 + 1, :], np.s_[:, w // 2 - 1:w // 2 + 1]]
    return [np.s_[h // 3 - 2:h // 3, :], np.s_[2 * h // 3:2 * h // 3 + 2, :],
            np.s_[:, w // 3 - 2:w // 3], np.s_[:, 2 * h // 3:2 * h // 3 + 2]]


def scalar_constants():
    """(OUTSIDE, ROAD, CAR, vocab) of vocab_type 'scalar' (:139-141): fixed classes, no BASE offset."""
    return 0, 1, 2, 2


def build_grid(difficulty, dim, vocab_type="bool"):
    """Road-id grid: every strip is numbered row-major in turn, later strips
    overwrite the junction cells; everything else is OUTSIDE.  vocab_type 'scalar'
    keeps the road-class grid instead (_set_grid :300-314 skips the numbering):
    ROAD = 1 on every strip, OUTSIDE = 0."""
    dims, _, outside, _, _, _ = constants(difficulty, dim)
    h, w = dims
    if vocab_type == "scalar":
        outside, road = scalar_constants()[:2]
        grid = np.full((h, w), outside, dtype=np.int64)
        for blk in road_blocks(h, w, difficulty):
            grid[blk] = road
        return grid
    grid = np.full((h, w), outside, dtype=np.int64)
    start = 0
    for blk in road_blocks(h, w, difficulty):
        shape = grid[blk].shape
        sz = int(np.prod(shape))
        grid[blk] = np.arange(start, start + sz).reshape(shape)
        start += sz
    return grid


def _junction_mask(h, w, difficulty):
    j = np.zeros((h, w), dtype=bool)
    if difficulty == "medium":
        j[h // 2 - 1:h // 2 + 1, w // 2 - 1:w // 2 + 1] = True
    elif difficulty == "hard":
        for rs in (slice(h // 3 - 2, h // 3), slice(2 * h // 3, 2 * h // 3 + 2)):
            for cs in (slice(w // 3 - 2, w // 3), slice(2 * w // 3, 2 * w // 3 + 2)):
                j[rs, cs] = True
    return j


def _arrivals(h, w, difficulty):
    if difficulty == "medium":
        return [((0, w // 2 - 1), DOWN), ((h - 1, w // 2), UP), ((h // 2, 0), RIGHT), ((h // 2 - 1, w - 1), LEFT)]
    return [((0, w // 3 - 2), DOWN), ((0, 2 * w // 3), DOWN),
            ((h // 3 - 1, 0), RIGHT), ((2 * h // 3 + 1, 0), RIGHT),
            ((h - 1, w // 3 - 1), UP), ((h - 1, 2 * w // 3 + 1), UP),
            ((h // 3 - 2, w - 1), LEFT), ((2 * h // 3, w - 1), LEFT)]


def _drive(start, heading, turns, junction):
    """Cells visited from ``start`` until the car leaves the map; also returns how
    many junctions were crossed."""
    h, w = junction.shape
    path = [start]
    r, c = start
    hd = heading
    met = 0
    inside = False      # currently on a junction block
    depth = 0           # junction cells driven on the current block
    turn = 0
    while True:
        nr, nc = r + hd[0], c + hd[1]
        if not (0 <= nr < h and 0 <= nc < w):
            return path, met
        r, c = nr, nc
        path.append((r, c))
        if junction[r, c]:
            if not inside:
                inside, depth = True, 0
                turn = turns[met] if met < len(turns) else 0
                met += 1
            depth += 1
            if turn == 1 and depth == 1:
                hd = _right_of(hd)
                turn = 0
            elif turn == 2 and depth == 2:
                hd = _left_of(hd)
                turn = 0
        else:
            inside = False


def build_routes(difficulty, dim):
    """list (arrival groups) of lists (paths) of [L,2] int arrays."""
    dims = constants(difficulty, dim)[0]
    h, w = dims
    if difficulty == "easy":
        return [[np.array([(i, w // 2) for i in range(h)], dtype=np.int64)],
                [np.array([(h // 2, i) for i in range(w)], dtype=np.int64)]]
    junction = _junction_mask(h, w, difficulty)
    n_turn2 = 1 if difficulty == "medium" else 3
    routes = []
    for start, heading in _arrivals(h, w, difficulty):
        paths = []
        for t1 in range(3):
            for t2 in range(n_turn2):
                path, met = _drive(start, heading, (t1, t2), junction)
                paths.append(np.array(path, dtype=np.int64))
                if met == 1:      # the first turn already led out of the map
                    break
        routes.append(paths)
    return routes


def build_tables(difficulty, dim, vision=0, vocab_type="bool"):
    """Everything the kernels need, as numpy arrays (uploaded once by the env).  The routes do not depend on
    vocab_type: both vocabularies hand get_routes the same road-class grid (:309,510)."""
    if vocab_type not in ("bool", "scalar"):
        raise ValueError("vocab_type must be 'bool' or 'scalar'")
    dims, base, outside, car, vocab, npath = constants(difficulty, dim)
    if vocab_type == "scalar":
        base = None
        outside, _, car, vocab = scalar_constants()
    if difficulty in ("easy", "medium"):          # traffic_junction_env.py:93-96
        assert dim % 2 == 0, "Only even dimension supported for now."
        assert dim >= 4 + vision, "Min dim: 4 + vision"
    if difficulty == "hard":                       # :98-100
        assert dim >= 9, "Min dim: 9"
        assert dim % 3 == 0, "Hard version works for multiple of 3. dim. only."
    grid = build_grid(difficulty, dim, vocab_type)
    routes = build_routes(difficulty, dim)
    G, P = len(routes), len(routes[0])
    assert all(len(g) == P for g in routes)
    assert G * P == npath                          # :520
    L = max(len(p) for g in routes for p in g)
    route_len = np.zeros((G, P), dtype=np.int32)
    route_cells = np.zeros((G, P, L), dtype=np.int32)
    for g, grp in enumerate(routes):
        for k, p in enumerate(grp):
            step = np.abs(np.diff(p, axis=0)).sum(1)
            assert np.all(step == 1)               # _unittest_path :526-537
            route_len[g, k] = len(p)
            route_cells[g, k, :len(p)] = (p[:, 0] << 16) | p[:, 1]
    return dict(dims=dims, BASE=base, OUTSIDE=outside, CAR=car, vocab=vocab, npath=npath, grid=grid,
                routes=routes, route_len=route_len, route_cells=route_cells, G=G, P=P, Lmax=L)
