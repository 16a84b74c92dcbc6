"""The poisoned-memory catalogue (tests/poison_cases.py) entry of borb_bow_score_batch: the case that drives it, registered in the
catalogue's CASES and COVERED tables when this module is imported.  A test run imports every test module before it runs any test,
so tests/test_poison_catalogue.py accounts for the entry point and tests/test_gpu_poison.py runs the case under 0x00, 0xFF and 0x7F
with the rest of the catalogue, after the keyframe-database case.  (tests/test_gpu_bow_score.py poisons the call on its own too.)"""
from tests import poison_cases as P
from tests.test_cabi import declared_symbols


def bow_score(c):
    """borb_bow_score_batch: frames and slots of two databases as queries and targets, a repeated target, a query among its own
    targets, and a job without targets."""
    M = c.M
    v, vs = c.big, c.small
    fr = [P._res(c, M.FrameView(x["kl"], x["dl"], x["scale"], (0.0, 0.0, float(x["w"]), float(x["h"])))) for x in (v, vs, v)]
    c.mt.ComputeBoWBatch(c.voc, fr, P.LEVELSUP, want_host=False)
    dbs = [M.KeyFrameDatabase(c.mt), M.KeyFrameDatabase(c.mt)]
    slots = c.mt.KfdbAddFramesBatch([dbs[0], dbs[1], dbs[0]], fr, None)
    sc = c.mt.BowScoreBatch([(fr[0], [(dbs[0], slots[0]), fr[1], (dbs[1], slots[1]), fr[1], fr[0]]),
                             ((dbs[0], slots[2]), [fr[2], (dbs[0], slots[0])]), (fr[1], [])])
    for F in fr:
        F.resident.close()
    return dict(slots=slots, sc=sc)


P.CASES.setdefault("bow_score", bow_score)
P.COVERED.setdefault("borb_bow_score_batch", ("bow_score",))


def test_catalogue_drives_bow_score():
    assert "borb_bow_score_batch" in declared_symbols()
    assert P.CASES["bow_score"] is bow_score and P.COVERED["borb_bow_score_batch"] == ("bow_score",)
    assert "borb_bow_score_batch" not in P.NOT_COVERED
