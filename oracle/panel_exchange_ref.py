"""oracle/panel_exchange_ref.py -- a small model of the per-column slot exchange of panel_getrf_kernel (csrc/panel.cu) on
grids of <= 32 CTAs, stepped through randomised interleavings on the CPU.

What is modelled (and nothing else: no arithmetic of the factorisation):
  * G CTAs, each two agents that meet at the CTA's block barriers: the ROW OWNERS (find the local candidate of column j,
    publish it, apply the rest of elimination j - 1) and the GATHER WARP (poll every CTA's header for column j, pick
    the winner, fetch the winner's row);
  * the slots: two parities x G CTAs x (4 header words + `nrow` row words), every word an "LL" word (payload, epoch)
    written and read ONE WORD AT A TIME, so a reader can see a slot that is half old, half new;
  * the epoch rule: column j of a launch with base b carries epoch b + j + 1 in slot parity j & 1; a reader spins until
    every word it needs carries that epoch;
  * the order inside a CTA, per column j:
        owners:  [rendezvous j-1]  candidate(j)  B1  publish(j)  B2  rest of elimination j-1   [rendezvous j]
        gather:  [rendezvous j-1]                B1              B2  gather(j)                 [rendezvous j]
    (column 0 has no B2).  `early_publish=True` moves the publish of the next column in front of the rendezvous, i.e. before
    this CTA's gather of the current column has finished: the order the kernel must never have.

run() raises ExchangeError when
  (i)   a slot word is overwritten before every CTA has finished the gather of the column the old word belonged to,
  (ii)  the agents stop making progress before every gather has completed (a spin that can never end), or
  (iii) two CTAs see a different winner or a different winner's row for some column."""
import random


class ExchangeError(AssertionError):
    pass


HDR = 4


def candidate(launch, g, j, nrow):
    """Deterministic stand-in for CTA g's candidate of column j: (key, pos, row) and its inner-block row."""
    h = (launch * 7919 + g * 104729 + j * 1299709) & 0xFFFFFFFF
    h = (h * 2654435761) & 0xFFFFFFFF
    key = h % 5                                     # few distinct keys: ties across CTAs are common
    pos = (h >> 8) % 1000 * 64 + g                  # unique per CTA
    row = g * 1000 + j
    return (key, pos, row), tuple((row, c) for c in range(nrow))


def better(a, b):
    return a[0] > b[0] or (a[0] == b[0] and a[1] < b[1])


class Model:
    def __init__(self, G, ncols, nrow=3, early_publish=False):
        assert 1 <= G <= 32
        self.G, self.ncols, self.nrow, self.early = G, ncols, nrow, early_publish
        # slots[par][g][word] = (payload, epoch, column tag for check (i))
        self.slots = [[[(None, 0, None)] * (HDR + nrow) for _ in range(G)] for _ in range(2)]
        self.epoch_base = 0                          # kept even, as the launcher does
        self.launch = 0

    # ---- one launch ----
    def run(self, rng):
        G, ncols = self.G, self.ncols
        self.gather_done = [-1] * G                 # last column whose gather CTA g has finished (this launch)
        self.seen = [[None] * ncols for _ in range(G)]
        self.bar = [dict() for _ in range(G)]       # per CTA: barrier name -> arrivals (two agents per CTA)
        agents = []
        for g in range(G):
            agents.append(self._owners(g))
            agents.append(self._gather(g))
        waiting = [None] * len(agents)              # None = runnable, ("bar", g, name) or ("spin", par, g, words, epoch)
        live = set(range(len(agents)))
        while live:
            ready = [i for i in sorted(live) if self._ready(waiting[i])]
            if not ready:
                raise ExchangeError("(ii) no progress: a gather can never complete")
            i = rng.choice(ready)
            try:
                waiting[i] = next(agents[i])
            except StopIteration:
                live.discard(i)
        for j in range(ncols):
            first = self.seen[0][j]
            for g in range(1, G):
                if self.seen[g][j] != first:
                    raise ExchangeError(f"(iii) column {j}: CTA 0 saw {first}, CTA {g} saw {self.seen[g][j]}")
        out = [self.seen[0][j] for j in range(ncols)]
        self.epoch_base += ncols + 2 + (ncols & 1)
        self.launch += 1
        return out

    def _ready(self, st):
        # a failed spin re-reads and changes nothing, so a spinning agent is only scheduled once its words carry the epoch
        if st is None:
            return True
        if st[0] == "bar":
            return self.bar[st[1]].get(st[2], 0) >= 2
        _, par, g, words, epoch = st
        return all(self.slots[par][g][w][1] == epoch for w in words)

    # ---- agents (generators; every yield is one interleaving point) ----
    def _barrier(self, g, name):
        self.bar[g][name] = self.bar[g].get(name, 0) + 1
        return ("bar", g, name)

    def _publish(self, g, j):
        epoch = self.epoch_base + j + 1
        par = j & 1
        cand, row = candidate(self.launch, g, j, self.nrow)
        words = [cand[0], 0, cand[1], cand[2]] + list(row)   # key (two words in the kernel), pos, row; then the row
        for w, payload in enumerate(words):
            old = self.slots[par][g][w]
            if old[2] is not None and old[2][0] == self.launch:
                oldcol = old[2][1]
                late = [c for c in range(self.G) if self.gather_done[c] < oldcol]
                if late:
                    raise ExchangeError(f"(i) CTA {g} overwrites word {w} of column {oldcol} with column {j} before "
                                        f"CTAs {late} finished that gather")
            self.slots[par][g][w] = (payload, epoch, (self.launch, j))
            yield None

    def _owners(self, g):
        published = -1
        for j in range(self.ncols):
            # candidate(j), B1
            yield self._barrier(g, ("B1", j))
            if published < j:
                yield from self._publish(g, j)
                published = j
            if j > 0:
                yield self._barrier(g, ("B2", j))
            yield None                              # rest of elimination j-1
            if self.early and j + 1 < self.ncols:
                # the forbidden order: the next column goes out before this CTA's gather of column j is known complete,
                # so nothing orders it after the other CTAs' gathers of column j - 1, whose slot parity it reuses
                yield from self._publish(g, j + 1)
                published = j + 1
            yield self._barrier(g, ("R", j))

    def _gather(self, g):
        for j in range(self.ncols):
            yield self._barrier(g, ("B1", j))
            if j > 0:
                yield self._barrier(g, ("B2", j))
            epoch = self.epoch_base + j + 1
            par = j & 1
            best, slot = None, -1
            for s in range(self.G):                  # the kernel polls one slot per lane; any order is allowed
                while True:
                    ws = []
                    for w in range(HDR):
                        ws.append(self.slots[par][s][w])
                    if all(x[1] == epoch for x in ws):
                        break
                    yield ("spin", par, s, tuple(range(HDR)), epoch)
                cand = (ws[0][0], ws[2][0], ws[3][0])
                if best is None or better(cand, best):
                    best, slot = cand, s
                yield None
            row = []
            for w in range(HDR, HDR + self.nrow):
                while self.slots[par][slot][w][1] != epoch:
                    yield ("spin", par, slot, (w,), epoch)
                row.append(self.slots[par][slot][w][0])
                yield None
            self.seen[g][j] = (best, tuple(row))
            self.gather_done[g] = j
            yield self._barrier(g, ("R", j))


def run(G, ncols, seed, launches=1, early_publish=False, nrow=3):
    """`launches` back-to-back launches on one set of slots (the epoch carries over); returns the winners per launch."""
    rng = random.Random(seed)
    m = Model(G, ncols, nrow=nrow, early_publish=early_publish)
    return [m.run(rng) for _ in range(launches)]


def expected(G, ncols, launch=0, nrow=3):
    out = []
    for j in range(ncols):
        best = None
        for g in range(G):
            cand, row = candidate(launch, g, j, nrow)
            if best is None or better(cand, best[0]):
                best = (cand, row)
        out.append(best)
    return out
