"""CHECKER ONLY — a plain numpy restatement of what filterGenotypes.py does per line: Genotype (genomics.py:317-356),
genomics.siteTest (742-799) and GenomeSite.asList (465-512), on the genotype tokens of one line.  The engine's
k_filter_sites / k_filter_thin / k_filter_emit are compared with it; the product never imports it.

A site is a list of (alleles, phase) tuples, one per selected sample in output order; populations are lists of indices into
it, in -p order."""
from __future__ import annotations

import numpy as np

DIPLO = dict(zip(("A", "C", "G", "K", "M", "N", "S", "R", "T", "W", "Y"),
                 ("AA", "CC", "GG", "GT", "AC", "NN", "CG", "AG", "TT", "AT", "CT")))
PAIR_DIPLO = {v: k for k, v in DIPLO.items()}
NUM = {"A": 0, "C": 1, "G": 2, "T": 3}


def genotype(tok, fmt, partial_to_missing=False):
    """(alleles, phase) of one token (Genotype.__init__ without the ploidy handling: widths are checked by the caller)"""
    if fmt == "phased":
        al = list(tok)[::2]
        ph = tok[1] if len(tok) > 1 and len(tok) % 2 == 1 else "/"
    elif fmt == "diplo":
        al, ph = list(DIPLO[tok]), "/"
    else:
        al, ph = list(tok), "/"
    if partial_to_missing and "N" in al:
        al = ["N"] * len(al)
    return tuple(al), ph


def is_missing(al):
    return any(a not in NUM for a in al)


def counts(gts, members=None):
    """A C G T counts over the non-missing alleles (binBaseFreqs(asCounts=True)); members None = every sample"""
    c = np.zeros(4, dtype=np.int64)
    for i in (range(len(gts)) if not members else members):
        for a in gts[i][0]:
            if a in NUM:
                c[NUM[a]] += 1
    return c


def freqs(c):
    n = c.sum()
    return np.array([np.nan] * 4) if n == 0 else 1. * c / n


def site_test(gts, pops, spec):
    """genomics.siteTest on one site.  spec: the keys of Engine.filter's spec (None / 0 = off)."""
    called = sum(not is_missing(al) for al, _ in gts)
    if called < spec.get("min_calls", 1):
        return False
    c = counts(gts)
    nal = int((c > 0).sum())
    if not spec.get("min_alleles", 1) <= nal <= spec.get("max_alleles", float("inf")):
        return False
    if nal > 1:
        if spec.get("min_var_count") and sorted(c)[-2] < spec["min_var_count"]:
            return False
        if spec.get("max_het") is not None:
            nhet = np.array([len(set(al)) > 1 for al, _ in gts]).sum()
            with np.errstate(divide="ignore", invalid="ignore"):
                h = 1. * nhet / np.int64(called)
            if h > spec["max_het"]:
                return False
        f2 = sorted(freqs(c))[-2]
        if spec.get("min_freq") and not spec["min_freq"] <= f2:
            return False
        if spec.get("max_freq") and not f2 <= spec["max_freq"]:
            return False
    if pops:
        if spec.get("min_pop_calls") is not None:
            for p, members in enumerate(pops):
                if sum(not is_missing(gts[i][0]) for i in members) < spec["min_pop_calls"][p]:
                    return False
        mpa, xpa = spec.get("min_pop_alleles"), spec.get("max_pop_alleles")
        if spec.get("fixed_diffs") or mpa is not None:
            by_pop = [set(np.flatnonzero(counts(gts, m) > 0)) for m in pops]
            if spec.get("fixed_diffs") and not (set(len(a) for a in by_pop) == {1} and len(set().union(*by_pop)) > 1):
                return False
            if mpa is not None:
                for p in range(len(pops)):
                    if not mpa[p] <= len(by_pop[p]) <= xpa[p]:
                        return False
        if spec.get("nearly_fixed_diff") is not None:
            pf = [freqs(counts(gts, m)) for m in pops]
            diffs = [pf[i] - pf[j] for i in range(len(pops)) for j in range(i + 1, len(pops))]
            with np.errstate(invalid="ignore"):
                if not np.any(np.absolute(np.concatenate(diffs)) >= spec["nearly_fixed_diff"]):
                    return False
    return True


def freq_order(c):
    """alleles by frequency, np.argsort(counts)[::-1] (genomics.py:556) with a stable sort"""
    idx = c > 0
    return list(np.array(["A", "C", "G", "T"])[idx][np.argsort(c[idx], kind="stable")[::-1]])


def is_tied(c):
    v = c[c > 0]
    return len(set(v.tolist())) < len(v)


def as_list(gts, mode, allele_order=None):
    """GenomeSite.asList(samples, mode, alleleOrder) as the strings filterGenotypes.py writes"""
    c = counts(gts)
    if mode in ("bases", "alleles"):
        if allele_order == "freq":
            order = freq_order(c) + ["N"]
            srt = [sorted(al, key=lambda x: order.index(x)) for al, _ in gts]
            return [a for s in srt for a in s] if mode == "bases" else ["".join(s) for s in srt]
        return [a for al, _ in gts for a in al] if mode == "bases" else [str(al) for al, _ in gts]
    if mode == "phased":
        return [ph.join(al) for al, ph in gts]
    if mode == "diplo":
        out = []
        for al, _ in gts:
            assert len(al) == 2, "Can only convert diploid genotypes to diplotypes."
            out.append(PAIR_DIPLO["".join(sorted(al))])
        return out
    order = freq_order(c)
    if mode == "coded":
        code = dict(zip(order, [str(x) for x in range(len(order))]))
        return [ph.join(["."] * len(al)) if is_missing(al) else ph.join(code[a] for a in al) for al, ph in gts]
    if mode == "count":
        target = order[-1]
        return [str(-1 if is_missing(al) else sum(a == target for a in al)) for al, _ in gts]
    raise ValueError(mode)


def filter_lines(lines, fmt, cols, pops, spec, out_mode, allele_order=None, include=None, exclude=None):
    """The whole worker loop of filterGenotypes.py:33-55 over data lines (the header excluded): lines in file order,
    cols = genotype column of every selected sample.  Returns the output rows (with their newline)."""
    out = []
    pod = spec.get("pod_size") or 10000
    thin = spec.get("thin_dist")
    last_scaf = last_pos = None
    for n, line in enumerate(lines):
        if n % pod == 0:
            last_scaf = None
        obj = line.split()
        if (include and obj[0] not in include) or (exclude and obj[0] in exclude):
            continue
        gts = [genotype(obj[2 + c], fmt, spec.get("partial_to_missing")) for c in cols]
        good = True
        if thin:
            pos = int(obj[1])
            if last_scaf != obj[0]:
                last_pos, last_scaf, good = pos, obj[0], False
            elif pos - last_pos < thin:
                good = False
        if good and not spec.get("no_test"):
            good = site_test(gts, pops, spec)
        if good:
            out.append("\t".join(obj[:2] + as_list(gts, out_mode, allele_order)) + "\n")
            if thin:
                last_pos = int(obj[1])
    return out
