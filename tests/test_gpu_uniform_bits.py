"""The varied-row stream's two row kinds (csrc/k1.cu uniform_prepare, k1_site_pass_packed<..., UNI>): a complete biallelic site
(every haplotype called, exactly two alleles: class byte 6 or 7 from csrc/ctx.cu k_pack_rows) is streamed as one plane,
"carries the higher of the two codes", any other varied site as three planes, and the uniform sites and every position are
added by k1_finalize from per-site prefixes.  Every record field (the popFreq columns included) must be bit-identical across
that stream, the stream with every varied row in three planes (PG_K1_UNI_BITS=0), the packed pass over every row
(PG_K1_NO_UNIFORM) and the byte pass (PG_K1_BYTE_PASS)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KNOBS = ("PG_K1_BYTE_PASS", "PG_K1_NO_UNIFORM", "PG_K1_UNIFORM_FORCE", "PG_K1_UNI_BITS", "PG_K1_UNI_R", "PG_K1_UNI_GV",
         "PG_K1_UNI_TMAX", "PG_K1_STAGES", "PG_K1_ACC_LIMIT")
PASSES = {"bits": {"PG_K1_UNIFORM_FORCE": "1"}, "planes": {"PG_K1_UNIFORM_FORCE": "1", "PG_K1_UNI_BITS": "0"},
          "packed": {"PG_K1_NO_UNIFORM": "1"}, "byte": {"PG_K1_BYTE_PASS": "1"}}
PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]     # A C G T: {A,T} and {C,G} differ in both code bits


@pytest.fixture(scope="module")
def eng():
    from genomics_general_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def _no_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def sites(rng, kinds, H):
    """one row per kind: 'u' uniform, 'm' all missing, 'b' complete biallelic (a random pair), 'b0' .. 'b5' biallelic of
    pair PAIRS[k], 't' biallelic plus a third allele in one haplotype, 'x' biallelic with one haplotype missing"""
    S = len(kinds)
    g = np.empty((S, H), np.int8)
    for s, k in enumerate(kinds):
        if k == "u":
            g[s] = rng.integers(0, 4)
        elif k == "m":
            g[s] = -1
        else:
            a, b = PAIRS[int(k[1]) if len(k) > 1 and k[0] == "b" else rng.integers(0, 6)]
            if H == 1:
                g[s] = a if k[0] != "m" else -1
                continue
            row = np.where(rng.random(H) < rng.random() * 0.8 + 0.1, b, a)
            row[rng.integers(0, H)] = a
            row[rng.integers(0, H)] = b if H > 1 else a
            if len(set(row.tolist())) < 2:
                row[0], row[-1] = a, b
            if k == "t":
                row[rng.integers(0, H)] = ({0, 1, 2, 3} - {a, b}).pop()
            elif k == "x":
                row[rng.integers(0, H)] = -1
            g[s] = row
    return g


def mixed(rng, S, H, frac=(0.55, 0.05, 0.3, 0.04, 0.06)):
    """uniform, all-missing, complete biallelic, third-allele and one-missing sites in the given shares"""
    kinds = rng.choice(["u", "m", "b", "t", "x"], S, p=frac)
    return sites(rng, kinds, H)


def layout(rng, H, P, interleaved):
    if interleaved:
        hp = (np.arange(H) % P).astype(np.int32)
        hp[rng.permutation(H)[:H // 10]] = -1
        for x in range(P):
            if not np.any(hp == x):
                hp[x] = x
        return hp
    cuts = np.sort(rng.choice(np.arange(1, H), P - 1, replace=False)) if P > 1 else np.zeros(0, np.int64)
    return np.repeat(np.arange(P), np.diff(np.concatenate([[0], cuts, [H]]))).astype(np.int32)


def set_knobs(monkeypatch, knobs):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv(k, str(v))


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def run(eng, monkeypatch, knobs):
    set_knobs(monkeypatch, knobs)
    out = []
    for freq in (False, True):
        eng.set_freqstats(freq)
        r = eng.popgen(2, 0.01)
        out.append((r, eng.popgen_freqstats() if freq else {}))
    eng.set_freqstats(False)
    return out, eng.uniform_stream()[0]


def stream_rows(eng, name):
    """the stream carries every complete biallelic site as one plane (none with PG_K1_UNI_BITS=0, nor at 5 to 8 populations,
    where the site pass walks three planes only), in the words that takes"""
    S, wd = eng.S, (eng.H + 31) // 32
    pw = (12 * wd + 15) // 16 * 4
    cls = eng.site_classes(0, S)
    varied = int(np.count_nonzero((cls == 0) | (cls >= 6)))
    one = int(np.count_nonzero(cls >= 6)) if name == "bits" and not 4 < eng.P <= 8 else 0
    n1, words = eng.uniform_rows()
    assert n1 == one, name
    assert one * wd + (varied - one) * pw <= words <= one * wd + (varied - one) * pw + 3 * eng.uniform_tiles()[2].size, name


def four_passes(eng, monkeypatch, knobs=None):
    """every record field of the four passes bit-identical; returns the records"""
    res = {}
    for name, pk in PASSES.items():
        res[name], used = run(eng, monkeypatch, dict(knobs or {}, **pk))
        assert used == (name in ("bits", "planes")), name
        if used:
            stream_rows(eng, name)
    for name in ("planes", "packed", "byte"):
        for (ra, fa), (rb, fb) in zip(res["bits"], res[name]):
            for k in ra:
                assert np.array_equal(bits(ra[k]), bits(rb[k])), (name, knobs, k)
            for k in fa:
                assert np.array_equal(bits(fa[k]), bits(fb[k])), (name, knobs, k)
    return res["bits"][0][0]


def upload_stale(eng, rng, g, pos):
    """g behind a wider matrix: an upload of its first rows zeroes them and 64 slack rows of the wider matrix's buffers, and
    the append of the rest, inside their capacity, lands on rows that keep the wider matrix's bytes past H"""
    S, H = g.shape
    eng.upload(rng.integers(0, 4, (S, H + 37)).astype(np.int8), np.arange(1, S + 1, dtype=np.int32))
    n0 = min(S, 10)
    eng.upload(g[:n0], pos[:n0])
    if S > n0:
        eng.append_sites(g[n0:], pos[n0:])


def load(eng, g, hp, P, lo, hi, pos=None, rng=None, stale=False):
    S = g.shape[0]
    if pos is None:
        pos = np.cumsum((rng or np.random.default_rng(0)).integers(1, 60, S)).astype(np.int32)
    if stale:
        upload_stale(eng, rng, g, pos)
    else:
        eng.upload(g, pos)
    eng.set_pops(hp, P)
    eng.set_windows(np.asarray(lo, np.int64), np.asarray(hi, np.int64))
    return pos


def windows(rng, S, w):
    lo = np.arange(0, S, w, dtype=np.int64)
    extra = rng.integers(0, S, 12)
    lo2 = np.concatenate([lo, extra, [0]])
    hi2 = np.minimum(np.concatenate([lo + w, extra + rng.integers(1, 3 * w, 12), [S]]), S)
    return lo2, hi2


def classes_np(g):
    """the class byte of each row, restated: 5 all missing, 1..4 one allele everywhere, 6 / 7 every haplotype called and two
    alleles that differ in the low bit only / in the high bit, else 0"""
    out = np.zeros(g.shape[0], np.uint8)
    for s, row in enumerate(g):
        called = row[row >= 0]
        al = sorted(set(called.tolist()))
        if called.size == 0:
            out[s] = 5
        elif called.size == row.size and len(al) == 1:
            out[s] = 1 + al[0]
        elif called.size == row.size and len(al) == 2:
            out[s] = 7 if (al[0] ^ al[1]) & 2 else 6
    return out


@pytest.mark.parametrize("H", [1, 31, 32, 33, 400, 1600])
def test_class_byte(eng, H):
    rng = np.random.default_rng(H)
    kinds = rng.choice(["u", "m", "b0", "b1", "b2", "b3", "b4", "b5", "t", "x"], 600)
    g = sites(rng, kinds, H)
    g[rng.random(600) < 0.05] = rng.integers(-1, 4, (1, H))        # anything at all
    upload_stale(eng, rng, g, np.arange(1, 601, dtype=np.int32))
    assert np.array_equal(eng.site_classes(0, 600), classes_np(g))


@pytest.mark.parametrize("H,P,inter", [(1, 1, False), (31, 3, True), (32, 2, False), (33, 5, True), (400, 4, False),
                                       (400, 8, True), (1600, 6, False), (1600, 3, True), (400, 7, True), (64, 1, False)])
def test_mixed_rows(eng, H, P, inter, monkeypatch):
    rng = np.random.default_rng(H * 10 + P)
    S = 6000
    g = mixed(rng, S, H) if H > 1 else sites(rng, rng.choice(["u", "m", "b"], S), 1)
    hp = layout(rng, H, P, inter) if H > 1 else np.zeros(1, np.int32)
    lo, hi = windows(rng, S, 500)
    load(eng, g, hp, P, lo, hi, rng=rng, stale=True)
    four_passes(eng, monkeypatch)


@pytest.mark.parametrize("kinds", ["b", "t", "u", "bt"])
def test_tile_kinds(eng, kinds, monkeypatch):
    """tiles with only one-plane rows, only three-plane rows, none (long uniform runs cut into pieces of Tmax), and each
    tile's one-plane rows and three-plane rows on either side of a segment boundary"""
    rng = np.random.default_rng(len(kinds) * 7 + ord(kinds[0]))
    S, H, P = 4000, 100, 4
    if kinds == "u":
        k = np.where(np.arange(S) % 1000 < 900, "u", "b")
    elif kinds == "bt":
        k = np.where(np.arange(S) % 16 < 8, "b", "t")          # 3-plane rows after one-plane rows in every tile
    else:
        k = np.where(rng.random(S) < 0.5, kinds, "u")
    g = sites(rng, k, H)
    hp = layout(rng, H, P, True)
    lo = np.arange(0, S, 12, dtype=np.int64)                  # segment edges inside every tile
    load(eng, g, hp, P, lo, np.minimum(lo + 12, S), rng=rng)
    four_passes(eng, monkeypatch, {"PG_K1_UNI_R": "32", "PG_K1_UNI_TMAX": "64"})
    four_passes(eng, monkeypatch, {"PG_K1_UNI_R": "40", "PG_K1_UNI_GV": "2"})


@pytest.mark.parametrize("knobs", [{"PG_K1_UNI_R": "7"}, {"PG_K1_UNI_R": "300"}, {"PG_K1_UNI_GV": "4"},
                                   {"PG_K1_UNI_GV": "32"}, {"PG_K1_STAGES": "2"}, {"PG_K1_ACC_LIMIT": "1"},
                                   {"PG_K1_UNI_TMAX": "8"}], ids=str)
def test_knobs(eng, knobs, monkeypatch):
    rng = np.random.default_rng(len(str(knobs)))
    S, H, P = 5000, 400, 4
    g = mixed(rng, S, H)
    lo, hi = windows(rng, S, 700)
    load(eng, g, layout(rng, H, P, False), P, lo, hi, rng=rng)
    four_passes(eng, monkeypatch, knobs)


@pytest.mark.parametrize("w,step", [(5000, 5000), (50000, 50000), (5000, 1000)])
def test_window_sizes(eng, w, step, monkeypatch):
    rng = np.random.default_rng(w + step)
    S, H, P = 120_000, 200, 4
    g = mixed(rng, S, H, (0.69, 0.01, 0.29, 0.01, 0.0))       # no partly missing site: the windows take the site pass
    lo = np.arange(0, S, step, dtype=np.int64) + 17
    hi = np.minimum(lo + w, S)
    load(eng, g, layout(rng, H, P, False), P, lo[lo < S], hi[lo < S], rng=rng)
    r = four_passes(eng, monkeypatch)
    assert np.count_nonzero(r["path"] == 1) > 0


def test_positions_and_appends(eng, monkeypatch):
    """a re-upload of the same genotypes with other positions, and appends, each followed by a popgen call: the position
    and uniform prefixes follow the data"""
    rng = np.random.default_rng(3)
    H, P = 60, 3
    g = mixed(rng, 3000, H)
    hp = layout(rng, H, P, True)
    eng.upload(rng.integers(0, 4, (5000, 80)).astype(np.int8), np.arange(1, 5001, dtype=np.int32))   # capacity
    pos = np.cumsum(rng.integers(1, 60, 3000)).astype(np.int64)

    def check(n, lo, hi):
        eng.set_windows(np.array(lo, np.int64), np.array(hi, np.int64))
        r = four_passes(eng, monkeypatch)
        assert list(r["pos_sum"]) == [int(pos[:n][a:b].sum()) for a, b in zip(lo, hi)]

    eng.upload(g[:1000], pos[:1000].astype(np.int32))
    eng.set_pops(hp, P)
    check(1000, [0, 300], [1000, 1000])
    pos[:1000] = pos[:1000] * 3 + 1
    eng.upload(g[:1000], pos[:1000].astype(np.int32))         # the same genotypes, other positions
    check(1000, [0, 300], [1000, 1000])
    pos[1000:] += pos[999]
    eng.append_sites(g[1000:2000], pos[1000:2000].astype(np.int32))     # inside the capacity
    check(2000, [0, 500, 1500], [2000, 1700, 2000])
    eng.append_sites(g[2000:], pos[2000:].astype(np.int32))
    check(3000, [0, 2500], [3000, 3000])
