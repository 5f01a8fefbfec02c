"""CPU tests of the sharded draw (tests/shard_draw.py): deterministic draws the restated refusal rule accepts, every
option covered by the suite's seeds, and the row cuts."""
from tests import shard_draw as D

REQUIRED = (
    ["loss 0", "loss 1"] + [f"mode {m}" for m in D.MODES] + [f"world {w}" for w in (2, 3, 4)]
    + [f"split {s}" for s in D.SPLITS]
    + ["column num", "column cat", "exact rule", "cat 256", "num 256", "gain hessian", "gain variance",
       "l1_regularization", "l2_regularization", "hessian_split_score_subtract_parent", "rng_words_consumed", "clamp",
       "min_examples 1", "min_examples 40", "in_split 0", "in_split 1", "sibling 0", "sibling 1", "depth 2", "depth 9",
       "depth 10", "weights", "best first", "drive step", "drive train"])


def test_every_draw_of_the_suite_is_accepted():
    for seed in list(D.SUITE_SEEDS) + [500, 777]:
        a, b = D.draw_sharded(seed), D.draw_sharded(seed)
        assert repr(a) == repr(b)
        assert D.refusal(a) is None, (seed, D.refusal(a))
        cuts = D.cuts(a)
        assert len(cuts) == a["world"]
        if a["mode"] != "features":
            assert cuts[0][0] == 0 and cuts[-1][1] == a["n"]
            assert all(c[1] == d[0] for c, d in zip(cuts, cuts[1:]))


def test_the_suite_covers_every_option():
    cov = D.coverage(D.SUITE_SEEDS)
    missing = [k for k in REQUIRED if k not in cov]
    assert not missing, f"not drawn by the suite's seeds: {missing}"


def test_the_refusals_are_restated():
    d = D.draw_sharded(0)
    for change, reason in ((dict(loss=2), "the multinomial loss is not combined with sharding"),
                           (dict(max_depth=10, sibling_subtraction=0), "more than 254 histogram slots")):
        assert D.refusal(dict(d, cfg=dict(d["cfg"], **change))) == reason
    cols = [dict(kind="num", B=8)] * 9
    assert D.refusal(dict(d, columns=cols, mode="rows_scatter", world=6, split="random")) is not None
    assert D.refusal(dict(d, columns=cols, mode="rows_scatter", world=5, split="random")) is None
    assert D.refusal(dict(d, columns=cols[:2], mode="features", world=3)) == "fewer features than ranks"
    assert D.refusal(dict(d, mode="rows", world=2, n=1, split="random")) == "a rank without rows"


def test_tiny_cuts_sit_around_the_row_block():
    d = dict(n=40000, world=4, mode="rows", split="tiny")
    assert [e - b for b, e in D.cuts(d)] == [1, 8191, 8192, 40000 - 16384]
