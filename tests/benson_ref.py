"""Benson's pass-alive chains and areas, restated in plain Python from the definition (include/elfb200.h,
elfb200_pass_alive), not from the kernel: breadth-first search over a list board.

stones: [N*N] by action a = x*N + y, 0 empty, 1 black, 2 white.  Returns (alive, area) as lists of N*N ints:
alive 1 on every stone of a pass-alive chain of either colour, area 1 / 2 on black's / white's pass-alive area."""


def neighbours(a, n):
    x, y = divmod(a, n)
    out = []
    if x > 0:
        out.append(a - n)
    if x < n - 1:
        out.append(a + n)
    if y > 0:
        out.append(a - 1)
    if y < n - 1:
        out.append(a + 1)
    return out


def components(points, n):
    """maximal 4-connected subsets of the set `points`, each a sorted list"""
    left, comps = set(points), []
    for a in sorted(points):
        if a not in left:
            continue
        comp, todo = {a}, [a]
        left.discard(a)
        while todo:
            for b in neighbours(todo.pop(), n):
                if b in left:
                    left.discard(b)
                    comp.add(b)
                    todo.append(b)
        comps.append(sorted(comp))
    return comps


def benson_colour(stones, n, c):
    """(alive stones, area points) of colour c, as sets"""
    P = n * n
    chains = components([a for a in range(P) if stones[a] == c], n)
    regions = components([a for a in range(P) if stones[a] != c], n)
    chain_of = {a: i for i, ch in enumerate(chains) for a in ch}
    libs = [set(b for a in ch for b in neighbours(a, n) if stones[b] == 0) for ch in chains]
    borders = [set(chain_of[b] for a in r for b in neighbours(a, n) if stones[b] == c) for r in regions]
    vital = []  # per region: the chains it is vital to
    for r in regions:
        empty = [a for a in r if stones[a] == 0]
        # a region without empty points would be opponent chains without liberties: not a legal position
        assert empty, "a region without empty points"
        v = set(i for i in range(len(chains)) if all(a in libs[i] for a in empty))
        # the vital chains are among the chains next to the region's first empty point
        assert v <= set(chain_of[b] for b in neighbours(empty[0], n) if stones[b] == c)
        vital.append(v)
    X, R = set(range(len(chains))), set(range(len(regions)))
    while True:
        x2 = set(i for i in X if sum(1 for r in R if i in vital[r]) >= 2)
        r2 = set(r for r in R if borders[r] <= x2)
        if x2 == X and r2 == R:
            break
        X, R = x2, r2
    alive = set(a for i in X for a in chains[i])
    area = set(a for r in R if vital[r] & X for a in regions[r])
    return alive, area


def benson(stones, n):
    stones = [int(s) for s in stones]
    alive, area = [0] * (n * n), [0] * (n * n)
    for c in (1, 2):
        al, ar = benson_colour(stones, n, c)
        for a in al:
            alive[a] = 1
        for a in ar:
            assert area[a] == 0, "the two colours' areas overlap"
            area[a] = c
    return alive, area
