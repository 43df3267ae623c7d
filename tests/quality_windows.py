"""
Quality-trimmed windows at their edges (test infrastructure only; reads neither the reference nor a device).

- ``scan`` / ``trim_index`` restate quality_trim_index (qualtrim.pyx:22-73) step by step, so that ``coverage`` can say
  which edges of the device's warp scan (cg_pscan.cuh, trim_scan_warp: 32 characters per step, the running maximum
  carried from step to step) a quality string reaches.  ``REQUIRED`` lists the edges the corpus
  tests/golden/qualtrim_edges_kat.json.gz (made by tests/golden/make_qualtrim_edges_golden.py) must hit.
- ``batch`` turns the corpus into read batches: warp compositions (whole tiles that need the warp scan, tiles where
  only lane 0 or lane 31 has a 256-character tail, empty reads, a ragged count, a shuffled copy) and reads whose
  adapter straddles an edge of the trimmed window with its missing part just outside (``poison``).
"""
import random

import numpy as np

from util import golden

TAILS = (0, 1, 31, 32, 33, 63, 64, 65, 96, 97, 128, 129, 255, 256)
CUTOFFS = ((0, 0), (0, 20), (5, 20), (20, 20), (40, 40), (60, 60), (25, 10))    # (25, 10): windows that meet
BASES = (33, 64)
NEXTSEQ_CUTOFFS = (20, 25)
ADAPTER = "AGATCGGAAGAGCACACGTCTGAACTCCAGTCA"
LINKED_BACK = "TGGAATTCTCGGGTGCCAAGG"


def code(c):
    """A quality character as both implementations read it: a signed char."""
    v = ord(c)
    return v - 256 if v >= 128 else v


def scan(q, cutoff, base, from_end):
    """One end of quality_trim_index: (partial sums in scan order, scan position of the first maximum or -1, position
    of the first negative sum or -1).  The scan stops at the first negative sum."""
    sums, best, first_max, neg = [], 0, -1, -1
    n = len(q)
    s = 0
    for k in range(n):
        s += cutoff - (code(q[n - 1 - k] if from_end else q[k]) - base)
        sums.append(s)
        if s < 0:
            neg = k
            break
        if s > best:
            best, first_max = s, k
    return sums, first_max, neg


def raw_trim(q, cf, cb, base):
    """(start, stop) before the window closes (qualtrim.pyx:71-72 not applied yet)."""
    n = len(q)
    _, m5, _ = scan(q, cf, base, False)
    _, m3, _ = scan(q, cb, base, True)
    return m5 + 1, n - 1 - m3 if m3 >= 0 else n


def trim_index(q, cf, cb, base):
    start, stop = raw_trim(q, cf, cb, base)
    return (0, 0) if start >= stop else (start, stop)


def nextseq_index(seq, q, cutoff, base):
    """nextseq_trim_index (qualtrim.pyx:76-117)"""
    s = best = 0
    stop = len(q)
    for i in reversed(range(len(q))):
        v = cutoff - 1 if seq[i] == "G" else code(q[i]) - base
        s += cutoff - v
        if s < 0:
            break
        if s > best:
            best, stop = s, i
    return stop


# ---- coverage -----------------------------------------------------------------------------------------------------

def _band(n):
    return "<=160" if n <= 160 else ("161-256" if n <= 256 else ">=257")


REQUIRED = (
    [f"tail{e}:{t}" for e in "53" for t in TAILS]
    + [f"length{e}:{b}" for e in "53" for b in ("<=160", "161-256", ">=257")]
    + [f"step{e}:{k}" for e in "53" for k in range(1, 9)]
    + [f"{kind}{e}:{what}" for e in "53" for kind, what in (
        ("max", "tie_next_step"), ("max", "lane0"), ("max", "lane31"), ("max", "last_character"),
        ("zero", "first"), ("zero", "run_across_step"), ("zero_then_negative", "lane0"),
        ("zero_then_negative", "lane31"), ("negative", "lane0"), ("negative", "lane31"))]
    + ["closed:bad_from_both_ends", "closed:meet", "closed:cross"]
    + [f"cutoff:{cf},{cb}:{b}" for cf, cb in CUTOFFS for b in BASES]
    + [f"below_base:{b}" for b in BASES] + ["byte>=128"]
    + [f"nextseq:{c}:{b}" for c in NEXTSEQ_CUTOFFS for b in BASES] + ["nextseq:window_tail>=32"]
)


def _end_keys(q, cutoff, base, e):
    sums, m, neg = scan(q, cutoff, base, e == "3")
    n = len(q)
    keys = set()
    keys.update(f"step{e}:{k}" for k in range(1, 9) if len(sums) > 32 * k)
    if m >= 0:
        best = sums[m]
        ties = [k for k, s in enumerate(sums) if s == best and (neg < 0 or k < neg)]
        if any(k // 32 == m // 32 + 1 for k in ties):
            keys.add(f"max{e}:tie_next_step")
        if m >= 32 and m % 32 == 0:
            keys.add(f"max{e}:lane0")
        if m >= 32 and m % 32 == 31:
            keys.add(f"max{e}:lane31")
        if m == n - 1 and n > 32:
            keys.add(f"max{e}:last_character")
    if n > 1 and sums[0] == 0:
        keys.add(f"zero{e}:first")
    if len(sums) > 33 and neg not in (31, 32) and sums[31] == sums[30] and sums[32] == sums[31]:
        keys.add(f"zero{e}:run_across_step")
    if neg >= 32 and neg % 32 in (0, 31):
        lane = "lane0" if neg % 32 == 0 else "lane31"
        keys.add(f"negative{e}:{lane}")
        if sums[neg - 1] == 0:
            keys.add(f"zero_then_negative{e}:{lane}")
    return keys


def entry_keys(q, cf, cb, base):
    """The edges one quality string reaches under (cf, cb, base)."""
    n = len(q)
    keys = {f"cutoff:{cf},{cb}:{base}"}
    keys |= _end_keys(q, cf, base, "5") | _end_keys(q, cb, base, "3")
    start, stop = raw_trim(q, cf, cb, base)
    if start < stop:
        for e, t in (("5", start), ("3", n - stop)):
            if t in TAILS and n > t:
                keys.add(f"tail{e}:{t}")
            if t >= 32:
                keys.add(f"length{e}:{_band(n)}")
    elif n:
        if start == n and stop == 0:
            keys.add("closed:bad_from_both_ends")
        elif start == stop:
            keys.add("closed:meet")
        else:
            keys.add("closed:cross")
    if any(code(c) < base for c in q):
        keys.add(f"below_base:{base}")
    if any(ord(c) >= 128 for c in q):
        keys.add("byte>=128")
    return keys


def coverage(corpus):
    """{edge: number of corpus entries that reach it}"""
    count = {}
    for fam, q, cf, cb, base, _, _ in corpus["quality"]:
        for k in entry_keys(q, cf, cb, base):
            count[k] = count.get(k, 0) + 1
    for fam, seq, q, ns_cut, cf, cb, base, ns_stop, start, stop in corpus["nextseq"]:
        if ns_stop < len(q):
            k = f"nextseq:{ns_cut}:{base}"
            count[k] = count.get(k, 0) + 1
        if start < stop and ns_stop - stop >= 32:
            count["nextseq:window_tail>=32"] = count.get("nextseq:window_tail>=32", 0) + 1
    return count


def missing(corpus):
    cov = coverage(corpus)
    return [k for k in REQUIRED if not cov.get(k)]


# ---- batches --------------------------------------------------------------------------------------------------------

def corpus():
    return golden("qualtrim_edges_kat.json.gz")


def pack(strings):
    """uint8 bytes (latin-1: quality bytes >= 128 stay single bytes) + int64 offsets."""
    joined = "".join(strings).encode("latin-1")
    offsets = np.zeros(len(strings) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in strings], out=offsets[1:])
    data = np.frombuffer(joined, dtype=np.uint8) if joined else np.zeros(1, dtype=np.uint8)
    return data, offsets


def param_sets(c):
    return sorted({(cf, cb, base) for _, _, cf, cb, base, _, _ in c["quality"]})


def _needs_warp_scan(q, cf, cb, base):
    """The first character of one end does not end that end's scan: the whole warp scans this read's tail."""
    return bool(q) and (cf - (code(q[0]) - base) >= 0 or cb - (code(q[-1]) - base) >= 0)


class Batch:
    """Reads of one parameter set: seqs, quals, their windows, and per read the poison layout (or None)."""

    def __init__(self, seqs, quals, windows, poison, params):
        self.seqs, self.quals, self.windows, self.poison, self.params = seqs, quals, windows, poison, params

    def __len__(self):
        return len(self.seqs)

    def packed(self):
        d, o = pack(self.seqs)
        q, _ = pack(self.quals)
        return d, o, q

    def fastq(self):
        """The batch as one FASTQ chunk (needs ASCII qualities)."""
        return "".join(f"@r{i}\n{s}\n+\n{q}\n" for i, (s, q) in enumerate(zip(self.seqs, self.quals))).encode("latin-1")


def _place(seq, lo, piece):
    """seq with piece written from index lo on (clipped to the read)."""
    seq = list(seq)
    for i, c in enumerate(piece):
        if 0 <= lo + i < len(seq):
            seq[lo + i] = c
    return seq


def poison(rng, seq, window, adapter, where):
    """The adapter straddles the window's end ('stop': its prefix ends the window, the rest follows outside) or its
    start ('start': its suffix starts the window, its prefix lies in front).  Returns (sequence, bytes of the adapter
    in front of the read that the previous read has to end with)."""
    s, e = window
    m = len(adapter)
    if where == "stop":
        k = rng.choice([3, 4, 5, m // 2, m - 2, m - 1])
        k = min(k, e - s)
        return "".join(_place(seq, e - k, adapter)), ""
    j = rng.choice([1, 1, 2, 3, m // 2])
    seq = _place(seq, s - j, adapter)
    return "".join(seq), adapter[:j - s] if s < j else ""


def batch(c, params, max_len=None, adapter=ADAPTER, seed=0, ascii_only=False, nextseq=False):
    """Reads of one parameter set (cf, cb, base), or with nextseq=True of one (nextseq cutoff, cf, cb, base), no longer
    than max_len, in the warp compositions and poisoned (see the module's doc)."""
    rng = random.Random(seed)
    if nextseq:
        ns_cut, cf, cb, base = params
        rows = [(seq, q, (s, e)) for _, seq, q, c_, f, b_, bs, _, s, e in c["nextseq"] if (c_, f, b_, bs) == params]
    else:
        cf, cb, base = params
        rows = [(None, q, (s, e)) for _, q, f, b_, bs, s, e in c["quality"] if (f, b_, bs) == (cf, cb, base)]
    rows = [r for r in rows if (max_len is None or len(r[1]) <= max_len)
            and (not ascii_only or all(33 <= ord(ch) < 127 for ch in r[1]))]
    assert rows, params
    warp = [r for r in rows if _needs_warp_scan(r[1], cf, cb, base)]
    long_tail = [r for r in rows if len(r[1]) >= 256 and (r[2][0] >= 255 or len(r[1]) - r[2][1] >= 255)]
    tiles = []
    tiles.append([warp[i % len(warp)] for i in range(32)] if warp else [])                  # every lane scans
    empty = (None, "", (0, 0))
    for lane in (0, 31):                                                                    # one lane scans 256
        if long_tail:
            t = [empty if i % 2 else (None, "I" * rng.randint(1, 9) if base == 33 else "h" * rng.randint(1, 9), None)
                 for i in range(32)]
            t[lane] = long_tail[lane % len(long_tail)]
            tiles.append(t)
    mixed = []
    for i, r in enumerate(rows):
        if i % 7 == 3:
            mixed.append(empty)
        mixed.append(r)
    order = [r for t in tiles for r in t] + mixed
    shuffled = list(order)
    rng.shuffle(shuffled)
    order = order + shuffled + order[:5]                                                    # count not % 32
    seqs, quals, windows, layout = [], [], [], []
    for seq, q, w in order:
        n = len(q)
        if w is None:
            w = trim_index(q, cf, cb, base) if not nextseq else None
        if seq is None:
            seq = "".join(rng.choice("ACGT") for _ in range(n))
        where = None
        # (with --nextseq-trim the bases after the window decide the window: the poison stays inside it)
        if w is not None and w[1] - w[0] >= (len(adapter) if nextseq else 3):
            where = "start" if nextseq else rng.choice(["stop", "start"])
            seq, before = poison(rng, seq, w, adapter, where)
            if before and seqs and len(seqs[-1]) >= len(before) and not nextseq:
                seqs[-1] = seqs[-1][: len(seqs[-1]) - len(before)] + before
        seqs.append(seq)
        quals.append(q)
        windows.append(w)
        layout.append(where)
    return Batch(seqs, quals, windows, layout, params)


def leaky_view(b, i):
    """The window of read i widened by the adapter's bytes just outside it: what a kernel that lets them in searches."""
    s, e = b.windows[i]
    seq = b.seqs[i]
    if b.poison[i] == "stop":
        return seq[s:min(len(seq), e + len(ADAPTER))]
    prev = b.seqs[i - 1] if i else ""
    mem = prev + seq
    lo = len(prev) + s
    return mem[max(0, lo - len(ADAPTER)):len(prev) + e]
