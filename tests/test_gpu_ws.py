"""windowStats on the H100: every fixture of tests/golden/ws13 through the device (byte for byte, zeros up to their sign), the
decimal parser against Python's float() bit for bit, the moments and order statistics against numpy at the pairwise tree's
split lengths, tiny chunks and sort budgets, and a large table against numpy."""
import math
import os
import struct

import numpy as np
import pytest

from test_ws_cpu import FAILS, OK, REFUSALS, TINY, case_args, expected, run_cli, same_up_to_zero_sign

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tiny", [False, True])
@pytest.mark.parametrize("case", OK, ids=[c["name"] for c in OK])
def test_device_matches_reference(case, tiny, tmp_path, monkeypatch):
    got = run_cli(case_args(case), tmp_path, monkeypatch, None, TINY if tiny else None)
    assert same_up_to_zero_sign(got, expected(case))


@pytest.mark.parametrize("case", FAILS, ids=[c["name"] for c in FAILS])
def test_device_refuses_before_any_output(case, tmp_path, monkeypatch):
    with pytest.raises(SystemExit) as e:
        run_cli(case_args(case), tmp_path, monkeypatch)
    assert REFUSALS[case["name"]] in str(e.value), str(e.value)
    assert run_cli.got == b""


def _tokens(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    bits = rng.integers(0, 1 << 63, n, dtype=np.int64).view(np.float64)
    for k in range(n):
        r = k % 10
        if r < 2:
            x = bits[k]
            out.append(repr(float(x)) if math.isfinite(x) else "1e-5")
        elif r == 2:
            out.append("%.*e" % (int(rng.integers(16, 25)), rng.random() * 10.0 ** int(rng.integers(-320, 308))))
        elif r == 3:
            d = "".join(map(str, rng.integers(0, 10, int(rng.integers(20, 800)))))
            p = int(rng.integers(0, len(d)))
            out.append(d[:p] + "." + d[p:] + "e%d" % int(rng.integers(-400, 400)))
        elif r == 4:
            out.append(rng.choice(["4.9e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "1e-400", "1e400",
                                   "2.2250738585072011e-308", "1.7976931348623158e308", "1.7976931348623159e308",
                                   "9007199254740993", "1_000.5", "1__0", "-0.0", "inf", "-nan", "0x1p3", "1d0", ".e1",
                                   "1e1_0", "_1", "1.5_", "+.5e-3"]))
        elif r == 5:                                                  # halfway between neighbours, printed exactly
            from decimal import Decimal
            x = float(rng.random() * 10.0 ** int(rng.integers(-20, 25)))
            out.append(format((Decimal(x) + Decimal(math.nextafter(x, math.inf))) / 2, "f"))
        elif r == 6:
            s = str(int(rng.integers(1, 1 << 62)))
            i = int(rng.integers(1, len(s)))
            out.append(s[:i] + "_" + s[i:] + "e-%d" % int(rng.integers(0, 30)))
        else:
            out.append("%.17g" % (rng.normal() * 10.0 ** int(rng.integers(-30, 30))))
    return out


def _load(eng, text):
    """one chunk, with the tokens the device leaves to the host resolved by float(), as the command line does"""
    S, _, _, fidx, ftok, err = eng.ws_chunk(text)
    assert err[0] == 0
    slot, line = np.divmod(fidx, S)
    st = (ftok & np.uint64(3)).astype(int)
    off = (ftok >> np.uint64(32)).astype(np.int64)
    ln = ((ftok >> np.uint64(2)) & np.uint64((1 << 30) - 1)).astype(np.int64)
    h = np.flatnonzero(st == 2)
    eng.ws_set_values(line[h], slot[h], [float(text[off[i]:off[i] + ln[i]]) for i in h])
    return S


def test_parser_matches_float_bit_for_bit():
    from genomics_general_b200.engine import Engine
    toks = _tokens(1_000_000, 11)
    text = "".join("c\t%d\t%s\n" % (i + 1, t) for i, t in enumerate(toks)).encode()
    with Engine(0) as eng:
        eng.ws_spec([0], 1, 1)
        S, _, _, fidx, ftok, err = eng.ws_chunk(text)
        assert S == len(toks) and err[0] == 0
        st = (ftok & np.uint64(3)).astype(int)
        line = fidx % S
        host = line[st == 2]
        eng.ws_set_values(host, np.zeros(len(host), np.int32), [float(toks[i]) for i in host])
        lo = np.arange(S, dtype=np.int64)
        vals, cnt = eng.ws_stats(lo, lo + 1, [2], [0.0], 1)                 # min of one value: the value itself
    rejected = set(line[st == 1].tolist())
    for i, t in enumerate(toks):
        try:
            want = float(t)
        except ValueError:
            assert i in rejected, t
            continue
        assert i not in rejected, t
        if math.isnan(want):
            assert cnt[i, 0] == 0, t
        else:
            assert struct.pack("<d", vals[i, 0, 0]) == struct.pack("<d", want), (t, vals[i, 0, 0], want)


SPLITS = [1, 2, 7, 8, 9, 15, 16, 17, 127, 128, 129, 136, 255, 256, 257, 264, 1000, 1024, 4095, 4097, 65536, 100000]


@pytest.mark.parametrize("budget", [1 << 30, 4096])
def test_moments_and_quantiles_match_numpy(budget):
    from genomics_general_b200.engine import Engine
    rng = np.random.default_rng(5)
    n = sum(SPLITS) + 1000
    v = rng.normal(0, 1, n) * 10.0 ** rng.integers(-4, 6, n)
    v[rng.random(n) < 0.1] = np.nan
    v[rng.random(n) < 0.001] = np.inf
    text = "".join("c\t%d\t%r\n" % (i + 1, float(x)) for i, x in enumerate(v)).encode()
    lo, hi, at = [], [], 0
    for k in SPLITS:                                  # windows of k non-NaN values, some overlapping
        idx = np.flatnonzero(~np.isnan(v[at:]))
        if len(idx) < k:
            break
        lo.append(at)
        hi.append(at + idx[k - 1] + 1)
        at = (at + hi[-1]) // 2
    stats = [0, 1, 2, 3, 4, 5, 6, 6, 6, 6, 6, 6]
    qs = [0, 0, 0, 0, 0, 0, 0.05, 0.1, 0.25, 0.75, 0.9, 0.95]
    with Engine(0) as eng:
        eng.ws_spec([0], 1, 1)
        _load(eng, text)
        vals, cnt = eng.ws_stats(np.array(lo), np.array(hi), stats, qs, 1, budget)
    import warnings
    for w, (a, b) in enumerate(zip(lo, hi)):
        x = v[a:b][~np.isnan(v[a:b])]
        assert cnt[w, 0] == len(x)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = [x.mean(), np.median(x), np.min(x), np.max(x), round(np.std(x), 6), np.sum(x)] + \
                [np.quantile(x, q) for q in qs[6:]]
        for k, wv in enumerate(want):
            g = vals[w, 0, k]
            assert (np.isnan(g) and np.isnan(wv)) or g == wv, (len(x), k, g, wv)


def test_large_table_against_numpy(tmp_path, monkeypatch):
    """2 * 10^6 lines of 4 columns through the command line with small chunks; every cell against numpy"""
    rng = np.random.default_rng(9)
    S = 2_000_000
    pos = np.cumsum(rng.integers(1, 20, S))
    M = rng.normal(0, 3, (S, 4))
    M[rng.random((S, 4)) < 0.05] = np.nan
    lines = ["s\tp\ta\tb\tc\td"] + ["chr\t%d\t%r\t%r\t%r\t%r" % (p, *map(float, r)) for p, r in zip(pos, M)]
    path = tmp_path / "big.tsv"
    path.write_text("\n".join(lines) + "\n")
    got = run_cli(["-i", str(path), "-w", "100000", "--stats", "mean", "sd", "median", "q90"], tmp_path, monkeypatch, None,
                  {"PG_WS_CHUNK_BYTES": str(16 << 20)})
    rows = got.decode().split("\n")[1:-1]
    bounds = np.searchsorted(pos, np.arange(0, pos[-1] + 100000, 100000) + 1)
    import warnings
    for k, row in enumerate(rows[:50] + rows[-5:]):
        w = k if k < 50 else len(rows) - 5 + (k - 50)
        a, b = bounds[w], bounds[w + 1]
        cells = row.split(",")[5:]
        for c in range(4):
            x = M[a:b, c][~np.isnan(M[a:b, c])]
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = [x.mean(), round(np.std(x), 6), np.median(x), np.quantile(x, 0.9)]
            assert cells[4 * c:4 * c + 4] == [str(np.float64(u)) for u in want], (w, c)
