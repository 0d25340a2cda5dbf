"""Host plumbing of the command lines that stream text through the device (parseVCF, filterGenotypes, genoToVCF, mergeGeno,
seqToGeno, genoToSeq, windowStats): the input is opened and its body cut into chunks of complete lines, the next chunk being
read (and decompressed) on a host thread while the device works on the current one; the device fills one pinned slab of
output while a host thread writes (and gzip-compresses) the other."""
from __future__ import annotations

import contextlib
import gzip
import io
import os
import re
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

EOL = re.compile(rb"\r\n|\r|\n")


def env_int(name, default):
    v = os.environ.get(name)
    return int(v) if v else default


def open_input(path):
    """a binary stream of the input: gzip for .gz, the file, or stdin when there is no path"""
    if not path:
        return sys.stdin.buffer
    return gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")


@contextlib.contextmanager
def open_output(path):
    """a binary stream of the output: gzip for .gz, the file, or sys.stdout.buffer when there is no path; closed (stdout
    flushed) on exit.  gzip's own default level 6: Python's default (9) compresses little better at a third of the speed."""
    out = (gzip.open(path, "wb", compresslevel=6) if path.endswith(".gz") else open(path, "wb")) if path \
        else sys.stdout.buffer
    try:
        yield out
    finally:
        if out is sys.stdout.buffer:
            out.flush()
        else:
            out.close()


def first_line(src):
    """(the first line, the bytes read after it) with universal newlines, as a text-mode readline reads it; None for an
    empty input"""
    buf = b""
    while True:
        m = EOL.search(buf)
        if m is not None and not (m.group() == b"\r" and m.end() == len(buf)):
            return buf[:m.start()], buf[m.end():]
        blk = src.read(1 << 16)
        if not blk:
            if not buf:
                return None
            return (buf[:m.start()], buf[m.end():]) if m is not None else (buf, b"")
        buf += blk


class Chain(io.RawIOBase):
    """the bytes already read from the stream, then the rest of it"""

    def __init__(self, head, stream):
        self.head, self.stream = head, stream

    def readable(self):
        return True

    def readinto(self, b):
        if self.head:
            n = min(len(b), len(self.head))
            b[:n] = self.head[:n]
            self.head = self.head[n:]
            return n
        data = self.stream.read(len(b))
        b[:len(data)] = data
        return len(data)


def chunks(stream, target, cut_at_cr=True):
    """Complete lines in chunks of about `target` bytes, cut after the last '\\n' or '\\r' (a '\\r\\n' cut in two leaves
    a blank line, which is skipped).  cut_at_cr=False cuts after the last '\\n' only, for callers to whom a blank line
    matters."""
    rest = b""
    eof = False
    while True:
        buf = rest
        while len(buf) < target and not eof:
            blk = stream.read(max(target - len(buf), 1))
            if not blk:
                eof = True
                break
            buf += blk
        if not buf:
            return
        if eof:
            yield buf
            return
        cut = max(buf.rfind(b"\n"), buf.rfind(b"\r") if cut_at_cr else -1) + 1
        if cut == 0:                        # one line longer than the target: read on
            blk = stream.read(target)
            if not blk:
                eof = True
            rest = buf + blk
            continue
        yield buf[:cut]
        rest = buf[cut:]


def prefetched(gen):
    """the items of gen, each read on a host thread while the caller works on the one before"""
    with ThreadPoolExecutor(1) as ex:
        fut = ex.submit(next, gen, None)
        while True:
            item = fut.result()
            if item is None:
                return
            fut = ex.submit(next, gen, None)
            yield item


def body_chunks(rest, src, target, cut_at_cr=True):
    """chunks() of the body (`rest`, the bytes read after the header, then the rest of src), prefetched"""
    return prefetched(chunks(io.BufferedReader(Chain(rest, src), buffer_size=1 << 20), target, cut_at_cr))


class SlabWriter:
    """Two slabs of `cap` bytes, each a `pinned((cap,), uint8)` (the engine's PinnedArray; the caller passes its own
    binding, so that a test can give a tool host arrays): the device fills one while a host thread hands the other to
    `write`.  slab() is the next free slab (its last write finished), write(nb) submits its first nb bytes, wait() blocks
    until every submitted write has finished.  On exit every write finishes before the slabs are freed; they are allocated
    on first use."""

    def __init__(self, write, cap, pinned):
        self._write, self.cap, self._pinned = write, cap, pinned
        self._bufs, self._pending, self._k = None, [None, None], 0
        self._ex = ThreadPoolExecutor(1)

    def slab(self):
        if self._bufs is None:
            self._bufs = [self._pinned((self.cap,), np.uint8) for _ in range(2)]
        if self._pending[self._k] is not None:
            self._pending[self._k].result()
        return self._bufs[self._k].array

    def write(self, nb):
        self._pending[self._k] = self._ex.submit(self._write, memoryview(self._bufs[self._k].array)[:nb])
        self._k ^= 1

    def wait(self):
        for f in self._pending:
            if f is not None:
                f.result()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        try:
            self.wait()
        finally:
            self._ex.shutdown()
            for b in self._bufs or ():
                b.close()
