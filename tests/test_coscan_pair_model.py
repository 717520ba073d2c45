"""A model of K1's pairs (scan_topk.cu: "pairs"): the tile tickets of a host's scan, the join kernel's jump on
the host's ticket counter, the guest-only wrap and the counter bookkeeping, played out over every interleaving
the test draws.  It checks the scheme the kernels implement: every tile is scored exactly once for the host and
exactly once for a joined guest, a refused guest scans every tile itself, and every counter ends where the
host-side bookkeeping says it does."""
import random

import pytest

TICKET_TILES = 4          # STB_TICKET_TILES
JUMP = 1 << 31            # STB_PAIR_JUMP
WARPS_PER_CTA = 8


def plan(tiles, warps):
    """stb_ticket_plan: bulk tickets of TICKET_TILES tiles, then the last ~2 tiles per warp one by one."""
    single = min(tiles, 2 * warps)
    t_bulk = (tiles - single) // TICKET_TILES
    n_tickets = t_bulk + (tiles - t_bulk * TICKET_TILES)
    return t_bulk, n_tickets


def ticket_tiles(t, t_bulk, off, tiles):
    t0 = t * TICKET_TILES if t < t_bulk else t_bulk * TICKET_TILES + (t - t_bulk)
    t1 = t0 + TICKET_TILES if t < t_bulk else t0 + 1
    return [(x + off) % tiles for x in range(t0, t1)]


def first_tile(t, t_bulk):
    return t * TICKET_TILES if t < t_bulk else t_bulk * TICKET_TILES + (t - t_bulk)


class Pair:
    def __init__(self, tiles, warps, off, t_base):
        self.tiles, self.warps, self.off = tiles, warps, off
        self.t_bulk, self.n_tickets = plan(tiles, warps)
        self.counter = t_base                  # the host's ticket counter
        self.t_base = t_base
        self.wrap = 0                          # the seat's wrap word (its tag: this launch)
        self.decided = None
        self.host = [0] * tiles
        self.guest = [0] * tiles

    def host_warp(self):
        """The ticket loop of a pair's host warp (stb_scan_q4, PAIR); yields before each atomic."""
        cur = yield "draw"
        while cur < JUMP and first_tile(cur, self.t_bulk) < self.tiles:
            nxt = yield "draw"                 # drawn before the ticket is scored
            for tile in ticket_tiles(cur, self.t_bulk, self.off, self.tiles):
                self.host[tile] += 1
            cur = nxt
        if cur < JUMP:
            return
        cur -= JUMP
        while first_tile(cur, self.t_bulk) < self.tiles:
            nxt = (yield "draw") - JUMP
            for tile in ticket_tiles(cur, self.t_bulk, self.off, self.tiles):
                self.host[tile] += 1
                self.guest[tile] += 1
            cur = nxt
        # the join kernel's decision (it writes it right after its add; the warp waits for it)
        if self.decided is None:
            return
        while True:
            w = yield "wrap"
            if w >= self.decided:
                break
            for tile in ticket_tiles(w, self.t_bulk, self.off, self.tiles):
                self.guest[tile] += 1

    def join(self, floor=0):
        """stb_pair_join_kernel: add the jump (after the host has drawn `floor`); the ticket the add returns is
        the join point, unless every ticket was drawn."""
        t = self.counter - self.t_base
        assert t >= floor or t >= self.n_tickets
        self.counter += JUMP
        self.decided = t if t < self.n_tickets else None
        return self.decided


def run(tiles, warps, join_step, seed, floor=0):
    """Plays one pair; join_step: the number of atomics the host's warps perform before the join kernel
    runs (None: no guest).  Returns the pair and the join result."""
    rng = random.Random(seed)
    p = Pair(tiles, warps, rng.randrange(tiles), t_base=rng.randrange(1 << 40))
    gens = [p.host_warp() for _ in range(warps)]
    pending = {i: next(g) for i, g in enumerate(gens)}
    steps, decided, tried = 0, None, False
    while pending:
        if join_step is not None and not tried and steps >= join_step:
            decided, tried = p.join(floor), True
        i = rng.choice(list(pending))
        op = pending[i]
        if op == "draw":
            val = p.counter - p.t_base
            p.counter += 1
        else:
            val = p.wrap
            p.wrap += 1
        steps += 1
        try:
            pending[i] = gens[i].send(val)
        except StopIteration:
            del pending[i]
    if join_step is not None and not tried:
        decided = p.join(floor)                # after the last draw: refused
    return p, decided


def grid_warps(tiles):
    """Warps of the grid a launch of `tiles` tiles gets on a small part (4 SMs x 2 CTAs x 8 warps)."""
    want = -(-tiles // WARPS_PER_CTA)
    return min(max(want, 1), 8) * WARPS_PER_CTA


@pytest.mark.parametrize("tiles", [1, 2, 7, 8, 63, 64, 65, 127, 128, 129, 132, 133, 300, 1001])
def test_every_tile_once_for_host_and_guest(tiles):
    warps = grid_warps(tiles)
    t_bulk, n_tickets = plan(tiles, warps)
    total = n_tickets + warps                  # atomics on the main counter: every warp draws once more
    # join positions: before the first draw, during the bulk tickets, in the one-by-one tail, after the last draw
    positions = sorted({0, 1, max(t_bulk // 2, 0), t_bulk, t_bulk + 1, (t_bulk + n_tickets) // 2, n_tickets - 1,
                        n_tickets, total, total + 5})
    for pos in positions:
        for seed in range(6):
            p, v = run(tiles, warps, pos, seed=1000 * tiles + 17 * pos + seed)
            assert p.host == [1] * tiles, (tiles, pos, seed)
            if v is not None:
                assert p.guest == [1] * tiles, (tiles, pos, seed, v)
                # the guest-only wrap is exactly the tiles before the join ticket
                assert sum(1 for t in range(v) for _ in ticket_tiles(t, t_bulk, 0, tiles)) == first_tile(v, t_bulk)
            else:
                assert p.guest == [0] * tiles          # refused: the guest's own scan reads everything
                assert pos >= n_tickets


@pytest.mark.parametrize("tiles", [5, 64, 129, 700])
def test_join_floor_delays_the_join_point(tiles):
    warps = grid_warps(tiles)
    _, n_tickets = plan(tiles, warps)
    floor = n_tickets // 2
    for seed in range(5):
        rng = random.Random(seed)
        p = Pair(tiles, warps, rng.randrange(tiles), t_base=rng.randrange(1 << 40))
        gens = [p.host_warp() for _ in range(warps)]
        pending = {i: next(g) for i, g in enumerate(gens)}
        v, joined = None, False
        while pending:
            if not joined and (p.counter - p.t_base >= floor or not pending):
                v, joined = p.join(floor), True   # the join kernel spins until the host has drawn `floor`
            i = rng.choice(list(pending))
            if pending[i] == "draw":
                val = p.counter - p.t_base
                p.counter += 1
            else:
                val = p.wrap
                p.wrap += 1
            try:
                pending[i] = gens[i].send(val)
            except StopIteration:
                del pending[i]
        if v is not None:
            assert v >= floor and p.guest == [1] * tiles
        else:
            assert p.guest == [0] * tiles
        assert p.host == [1] * tiles


def test_booked_counters_match_the_device_counters():
    """The host books each launch's advance before it runs: n_tickets + warps, plus the jump on a host's counter
    when a guest launches, which the join kernel adds; the joined guest's scan kernel adds its own booking."""
    rng = random.Random(7)
    for _ in range(200):
        tiles = rng.randrange(1, 2000)
        warps = grid_warps(tiles)
        _, n_tickets = plan(tiles, warps)
        total = n_tickets + warps
        has_guest = rng.random() < 0.8
        pos = rng.randrange(0, total + 3) if has_guest else None
        p, v = run(tiles, warps, pos, seed=rng.randrange(1 << 30))
        booked_host = p.t_base + n_tickets + warps + (JUMP if has_guest else 0)
        assert p.counter == booked_host        # the join adds the jump once, joined or not
        if has_guest and v is None:
            # a refused guest's scan kernel scans alone and draws exactly its booking (joined, its first CTA
            # adds the booking in one atomic)
            g_base = rng.randrange(1 << 40)
            booked_guest = g_base + n_tickets + warps
            q = Pair(tiles, warps, 0, g_base)
            gens = [q.host_warp() for _ in range(warps)]
            pending = {i: next(g) for i, g in enumerate(gens)}
            while pending:
                i = rng.choice(list(pending))
                val = q.counter - q.t_base
                q.counter += 1
                try:
                    pending[i] = gens[i].send(val)
                except StopIteration:
                    del pending[i]
            assert q.host == [1] * tiles and q.counter == booked_guest
