#!/usr/bin/env python
"""Generate the agari (winning-hand decomposition) table from first principles -- no input files.

What the table is (format: SURVEY.md Appendix A; consumer: libriichi/src/algo/agari.rs:22-51, 126-157, 767-838):
a hand of 3n+2 concealed tiles is abstracted to its *shape*: the sequence of maximal runs of adjacent tile kinds
("blocks"; honours are blocks of length one) with the count of every kind.  `shape_key` below is that abstraction as
the reference computes it (agari.rs:767-838).  The table maps the key of every shape that splits into n melds and
one pair (n = 0..4), or into seven distinct pairs, to the list of its splits ("divs"), each one u32:

    bits 0-2  number of triplets      bits 3-5  number of runs      bits 6-9  index of the pair
    bits 10.. 4-bit indices of the triplets, then of the runs (index of a run = index of its lowest tile)
    bit 26 seven pairs   bit 27 nine gates   bit 28 straight 1-9   bit 29 two double runs   bit 30 one double run

where an index counts the distinct kinds of the hand in ascending order (`tile14`).

Enumeration: a block is any run that occurs when <= 4 melds and <= 1 pair are laid into one suit; a shape is any
sequence of blocks holding exactly one pair and <= 4 melds (the number of melds / pairs of a block follows from its tile
count).  Splits are listed per pair position (ascending) by a depth-first search that tries a triplet before a run at
every kind.  Three details are properties of the published table rather than of mahjong, and are kept because the
table's content is part of the contract (the oracle and the CUDA library must see what libriichi sees):

* four adjacent triplets `aaa bbb ccc ddd` list {4 triplets} and {abc abc abc + ddd} but not {aaa + bcd bcd bcd};
* the double-run flags are only set on four-meld (14-tile) splits (agari.rs:61-62 "sound but not complete");
* a seven-pairs shape that also splits into melds (two double runs) carries no seven-pairs flag.

File order: ascending key (the reference loads its file into a hash map, so the order of its records is not content).
`tests/test_tables.py` compares key -> ordered div list with libriichi's data file (tests/golden/tables/agari.bin.gz).
"""
import itertools
import struct
import sys
from collections import Counter

F_CHITOI, F_CHUUREN, F_ITTSUU, F_RYANPEIKOU, F_IPEIKOU = (1 << b for b in range(26, 31))


def shape_key(blocks) -> int:
    """agari.rs:767-838 on the abstract shape: per kind one position bit, a count code above it (2 -> 11, 3 -> 1111,
    4 -> 111111), and a set bit where the run ends."""
    key, bit = 0, -1
    for block in blocks:
        for c in block:
            bit += 1
            if c >= 2:
                width = 2 * (c - 1)
                key |= ((1 << width) - 1) << bit
                bit += width
        key |= 1 << bit
        bit += 1
    return key


def block_types():
    """Every run of adjacent kinds that <= 4 melds plus <= 1 pair can form inside one suit."""
    melds = [("k", i) for i in range(9)] + [("s", i) for i in range(7)]
    found = set()
    for n in range(5):
        for combo in itertools.combinations_with_replacement(melds, n):
            base = [0] * 9
            for kind, i in combo:
                if kind == "k":
                    base[i] += 3
                else:
                    for j in range(3):
                        base[i + j] += 1
            for pair in [None] + list(range(9)):
                counts = list(base)
                if pair is not None:
                    counts[pair] += 2
                if max(counts) > 4:
                    continue
                run = []
                for c in counts + [0]:
                    if c:
                        run.append(c)
                    elif run:
                        found.add(tuple(run))
                        run = []
    return sorted(found)


def shapes(blocks):
    """All block sequences with exactly one pair and at most four melds."""
    cost = {b: divmod(sum(b), 3) for b in blocks}  # (melds, 2 if the block holds the pair else 0)
    out, seq = [], []

    def rec(melds, has_pair):
        if has_pair:
            out.append(tuple(seq))
        for b in blocks:
            m, r = cost[b]
            if melds + m <= 4 and not (has_pair and r):
                seq.append(b)
                rec(melds + m, has_pair or r == 2)
                seq.pop()

    rec(0, False)
    return out


def splits(shape):
    """[(pair idx, triplet idxs, run idxs)] in table order."""
    counts = [c for b in shape for c in b]
    adj = [j + 1 < len(b) for b in shape for j in range(len(b))]  # kind i+1 is adjacent to kind i
    n = len(counts)
    out = []

    def rec(i, c, ks, ss, acc):
        while i < n and c[i] == 0:
            i += 1
        if i == n:
            acc.append((tuple(ks), tuple(ss)))
            return
        if c[i] >= 3:
            c[i] -= 3
            ks.append(i)
            rec(i, c, ks, ss, acc)
            ks.pop()
            c[i] += 3
        if i + 2 < n and adj[i] and adj[i + 1] and c[i + 1] and c[i + 2]:
            for j in range(3):
                c[i + j] -= 1
            ss.append(i)
            rec(i, c, ks, ss, acc)
            ss.pop()
            for j in range(3):
                c[i + j] += 1

    for pair in range(n):
        if counts[pair] < 2:
            continue
        c = list(counts)
        c[pair] -= 2
        acc = []
        rec(0, c, [], [], acc)
        for ks, ss in acc:
            if len(ks) == 1 and ss == (ks[0] + 1,) * 3 and adj[ks[0]]:
                continue  # aaa + bcd bcd bcd of four adjacent triplets: absent from the published table
            if (pair, ks, ss) not in out:
                out.append((pair, ks, ss))
    return out


def encode(shape, pair, ks, ss) -> int:
    v = len(ks) | len(ss) << 3 | pair << 6
    for j, idx in enumerate(ks + ss):
        v |= idx << (10 + 4 * j)
    start, length, i = [], [], 0
    for b in shape:
        start += [i] * len(b)
        length += [len(b)] * len(b)
        i += len(b)
    if len(shape) == 1 and len(shape[0]) == 9 and sum(shape[0]) == 14 and shape[0][0] >= 3 and shape[0][8] >= 3:
        v |= F_CHUUREN
    if any(length[s] == 9 and s == start[s] and s + 3 in ss and s + 6 in ss for s in ss):
        v |= F_ITTSUU
    if len(ks) + len(ss) == 4:
        doubles = sum(cnt // 2 for cnt in Counter(ss).values())
        if len(ss) == 4 and doubles == 2:
            v |= F_RYANPEIKOU
        elif doubles:
            v |= F_IPEIKOU
    return v


def generate() -> dict:
    """key -> [div, ...]"""
    table = {}
    for shape in shapes(block_types()):
        key = shape_key(shape)
        assert key not in table
        divs = [encode(shape, *s) for s in splits(shape)]
        assert 1 <= len(divs) <= 4
        table[key] = divs
    # seven distinct pairs; each of the six gaps between consecutive pairs is "adjacent" or not
    for gaps in itertools.product((False, True), repeat=6):
        shape = [[2]]
        for adjacent in gaps:
            if adjacent:
                shape[-1].append(2)
            else:
                shape.append([2])
        table.setdefault(shape_key(shape), [F_CHITOI])
    return table


def serialize(table: dict) -> bytes:
    out = bytearray()
    for key in sorted(table):
        out += struct.pack("<IB", key, len(table[key]))
        out += struct.pack(f"<{len(table[key])}I", *table[key])
    return bytes(out)


def parse(raw: bytes) -> dict:
    table, p = {}, 0
    while p < len(raw):
        key, n = struct.unpack_from("<IB", raw, p)
        table[key] = list(struct.unpack_from(f"<{n}I", raw, p + 5))
        p += 5 + 4 * n
    return table


if __name__ == "__main__":
    data = serialize(generate())
    if len(sys.argv) > 1:
        with open(sys.argv[1], "wb") as f:
            f.write(data)
    print(f"agari table: {len(parse(data))} keys, {len(data)} bytes")
