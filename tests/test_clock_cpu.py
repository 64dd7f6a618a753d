"""The referenced-key spec of CLOCK mode (tests/clock_oracle.py) on hand-made cases."""
from oracle import kvoracle as ko
from clock_oracle import referenced_keys, walk_keys

B = 4
TP = ko.ChunkedTokenDatabase(B)


def prompt(n_blocks, salt=0):
    return [1000 * salt + j for j in range(n_blocks * B)]


def keys_of(tokens, model="m"):
    return TP.tokens_to_kv_block_keys(None, tokens, model)


def index_with(keys_pods, model="m"):
    """keys_pods: [(Key, [pod, ...]), ...] -> InMemoryIndex holding them (engine key = request key)."""
    ix = ko.InMemoryIndex(1 << 20, 10)
    for k, pods in keys_pods:
        ix.add([k], [k], [ko.PodEntry(p, "gpu") for p in pods])
    return ix


def test_gap_at_block_i():
    t = prompt(6)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for j, k in enumerate(ks) if j != 3])
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set(ks[:3])


def test_filter_empties_active_set_early():
    t = prompt(5)
    ks = keys_of(t)
    ix = index_with([(ks[0], ["a", "b"]), (ks[1], ["a", "b"]), (ks[2], ["b"]), (ks[3], ["a"]), (ks[4], ["a"])])
    # unfiltered: block 2 keeps b, block 3 drops it -> blocks 0..3
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set(ks[:4])
    # filter {a}: block 2 holds only b -> the walk ends at block 2
    assert referenced_keys(ix, [(t, "m")], [["a"]], block_size=B) == set(ks[:3])


def test_key0_absent():
    t = prompt(4)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks[1:]])
    assert referenced_keys(ix, [(t, "m")], block_size=B) == set()


def test_present_but_filtered_out_counts_as_probed():
    t = prompt(3)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks])
    assert referenced_keys(ix, [(t, "m")], [["b"]], block_size=B) == {ks[0]}
    # the same at block 1: block 1 is probed (and marked), block 2 is not
    ix2 = index_with([(ks[0], ["a", "b"]), (ks[1], ["a"]), (ks[2], ["a", "b"])])
    assert referenced_keys(ix2, [(t, "m")], [["b"]], block_size=B) == {ks[0], ks[1]}


def test_several_models():
    t = prompt(3)
    ka, kb = keys_of(t, "A"), keys_of(t, "B")
    ix = index_with([(k, ["p"]) for k in ka] + [(kb[0], ["p"])])
    got = referenced_keys(ix, [(t, "A"), (t, "B")], block_size=B)
    assert got == set(ka) | {kb[0]}
    assert referenced_keys(ix, [(t, "B")], block_size=B) == {kb[0]}


def test_walk_does_not_refresh_recency():
    t = prompt(3)
    ks = keys_of(t)
    ix = index_with([(k, ["a"]) for k in ks])
    before = list(ix.data.d)
    assert walk_keys(ix, ks) == ks
    assert list(ix.data.d) == before
