"""Derives the tables `fold_coef` of csrc/cfr_board.cu: for a compiled post-deal shape of Flop5Holdem, the opponent's reach at
every FOLD terminal as a +-1 combination of its reach at the SHOWDOWN terminals (the opponent's strategies sum to one at its
own nodes, the sweep's seat copies the reach at its nodes).  The sweep kernel uses it to get the card-row sums of the fold
vectors from the showdown vectors' row totals instead of gathering them (update form).

    python tools/fold_relations.py        # prints the table of ShapeFHP in the C initialiser's layout
    python tools/fold_relations.py 1,0,0,4,1,3,4,3,4 1,3,5,-1,7,-1,-1,-1,-1 2,2,2,0,2,0,0,0,0
                                          # ... of the shape with these kind / first_child / n_children arrays (ShapeFHPShort)

Method: random strategies -> reach of the opponent at every node -> least squares of each fold vector on the showdown
vectors; the residual must vanish and the coefficients must be integers."""
import numpy as np

# ShapeFHP of csrc/cfr_board.cu (breadth-first): kind 0 / 1 = seat to act, 3 = fold terminal, 4 = showdown terminal
KIND = [1, 0, 0, 4, 1, 3, 4, 1, 3, 4, 0, 3, 4, 3, 4]
FIRST = [1, 3, 5, -1, 8, -1, -1, 11, -1, -1, 13, -1, -1, -1, -1]
NCH = [2, 2, 3, 0, 3, 0, 0, 2, 0, 0, 2, 0, 0, 0, 0]


def derive(kind=KIND, first=FIRST, nch=NCH, trials=40, seed=0):
    """int [2 seats][n_fold][n_sd] (seat = the seat whose values the sweep computes; the reach is its opponent's)"""
    n = len(kind)
    sd = [i for i in range(n) if kind[i] == 4]
    fo = [i for i in range(n) if kind[i] == 3]
    rng = np.random.default_rng(seed)
    out = np.zeros((2, len(fo), len(sd)), np.int64)
    for seat in (0, 1):
        opp = 1 - seat
        X = np.zeros((trials, n))
        for t in range(trials):
            x = np.zeros(n)
            x[0] = rng.random() + 0.1
            for i in range(n):
                if kind[i] <= 1:
                    s = np.ones(nch[i])
                    if kind[i] == opp:
                        s = rng.random(nch[i]) + 0.05
                        s /= s.sum()
                    for c in range(nch[i]):
                        x[first[i] + c] = x[i] * s[c]
            X[t] = x
        for k, f in enumerate(fo):
            coef, *_ = np.linalg.lstsq(X[:, sd], X[:, f], rcond=None)
            assert np.abs(X[:, sd] @ coef - X[:, f]).max() < 1e-12, "fold vector %d is not in the span of the showdown vectors" % f
            assert np.abs(coef - np.round(coef)).max() < 1e-9
            out[seat, k] = np.round(coef).astype(np.int64)
    return out


def as_c_initialiser(tab):
    return "{" + ", ".join("{" + ", ".join("{" + ", ".join(str(int(v)) for v in row) + "}" for row in seat) + "}" for seat in tab) + "}"


if __name__ == "__main__":
    import sys
    if len(sys.argv) == 4:
        print(as_c_initialiser(derive(*([int(x) for x in a.split(",")] for a in sys.argv[1:]))))
    else:
        print(as_c_initialiser(derive()))
