"""GPU (-m gpu): the class pipeline keeps its live list in batch order from round to round.

The round-0 list is sorted by first-block fingerprint, so the members of a prefix class are list neighbours, and kernel G
takes a neighbour whose chunk equals the running anchor's without the election (whose losers read two chunks again).
If the next round's list keeps the order of this one, that holds in every round: a class then only goes through the
election more than once where it straddles one of G's 32-prompt tiles, so a round has at most one election loser per
tile.  A list rebuilt in any other order separates class-mates and shows up as a loser for almost every class.  The
counts come from the KVIDX_ROUNDS_TRACE=1 line of every round and part; the scores are checked against the oracle."""
import math
import re

import numpy as np
import pytest

from helpers import _index_pair, _select_path, csr

pytestmark = pytest.mark.gpu
BS = 16
TRACE = re.compile(r"round (\d+) part (\d+): live (\d+) .*?; G streamed (\d+) chunks, (\d+) losers re-read")


@pytest.mark.parametrize("path", ["classes", "classes8"])
def test_next_live_list_keeps_batch_order(monkeypatch, capfd, path):
    _select_path(monkeypatch, path)
    monkeypatch.setenv("KVIDX_ROUNDS_TRACE", "1")
    ix, co = _index_pair(capacity=1 << 17, max_pods=64)
    rng = np.random.default_rng(11)
    distinct, copies, blocks = 400, 3, 4 * 32          # classes of three that stay together for four rounds
    base = [rng.integers(0, 50000, size=blocks * BS, dtype=np.uint32) for _ in range(distinct)]
    for d, b in enumerate(base):                        # every block is cached (on one pod), so no walk ends early
        keys = ix.hash_keys(b, np.array([0, len(b)], np.int64))[0]
        assert len(keys) == blocks
        eng = (keys ^ np.uint64(0x77)).astype(np.uint64)
        pt = [(d % 64) << 4]
        assert ix.add(0, eng, keys, pt) == 0
        co.add(0, eng, keys, pt)
    order = rng.permutation(distinct * copies) % distinct
    tok, off = csr([base[i] for i in order])
    capfd.readouterr()
    s_t, h_t = ix.score_batch(tok, off)
    err = capfd.readouterr().err
    s_o, h_o, _, _ = co.score_batch(tok, off, n_threads=4)
    assert np.array_equal(h_t, h_o) and np.array_equal(s_t, s_o)
    rows = [tuple(int(v) for v in m.groups()) for m in TRACE.finditer(err)]
    assert rows, err
    later = [r for r in rows if r[0] >= 1 and r[2] > 0]
    assert {r[0] for r in later} == {1, 2, 3}, err       # the classes live on for three more rounds
    for rnd, part, live, streamed, losers in rows:
        assert streamed == live, (rnd, part, err)
        # (round 0 also counts losers of map-bucket collisions between different prompts, which pass the metadata check
        # there; from round 1 on, different classes have different chain states and never get as far as the tokens)
        if rnd >= 1:
            assert losers <= math.ceil(live / 32), (rnd, part, live, losers)
