"""CPU tests of the ground-truth seeding and the hungarian association in the tracker restatement
(oracle/tracker_ref.py): restatement == golden (tests/golden/tracker_seq_{gt_first,gt_every,hungarian}.json, from the
unmodified reference through oracle/make_golden_tracker_gt.py) == the live reference when its tree is present; and the
option defaults of default_opt() equal the reference's parsed defaults."""
import json
import os
import types

import pytest

import centerpose_b200 as cpb
from oracle import make_golden_tracker_gt as mgt
from oracle import pnp_ref, ref_shims, tracker_ref
from tests.test_oracle_tracker import _compare

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _restatement(gold_opt, name):
    opt = types.SimpleNamespace(**{k: v for k, v in gold_opt.items() if k != "conf_border"})
    opt.conf_border = {opt.c: gold_opt["conf_border"]}

    def shell(det, pts, meta):
        return pnp_ref.pnp_shell(det, pts, meta["camera_matrix"], meta["width"], meta["height"], category=opt.c,
                                 opencv_return=opt.show_axes)[1]
    return mgt.run_scenario(name, tracker_ref.TrackerRef, shell, tracker_ref.gaussian_fusion, opt)


@pytest.mark.parametrize("name", mgt.SCENARIOS)
def test_restatement_matches_reference_golden(name):
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_%s.json" % name)))
    assert gold["scenario"] == name and bool(gold["opt"]["hungarian"]) == (name == "hungarian")
    _compare(_restatement(gold["opt"], name), gold["frames"])
    ids = [[t["tracking_id"] for t in fr["tracks"]] for fr in gold["frames"]]
    if name != "hungarian":
        assert ids[0] == [1, 2, 3, 4, 5]                 # five seeds above new_thresh; the 0.2 seed starts nothing
    if name == "gt_first":
        ages = {t["tracking_id"]: t["age"] for t in gold["frames"][0]["tracks"]}
        assert ages[4] == 2 and ages[5] == 2             # seeds without a detection are lost, not dropped
        assert max(max(i) for i in ids) == 6             # a new object after the seeds gets the next id
    if name == "gt_every":
        assert all(i[:3] == [1, 2, 3] for i in ids)      # ids restart at every re-seeding


@pytest.mark.skipif(not ref_shims.reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("name", mgt.SCENARIOS)
def test_golden_is_what_the_live_reference_computes(name):
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_%s.json" % name)))
    _compare(mgt.run_reference(name)["frames"], gold["frames"])


def test_hungarian_changes_the_association():
    gold = json.load(open(os.path.join(GOLDEN, "tracker_seq_hungarian.json")))
    greedy = dict(gold["opt"], hungarian=False)
    ids = lambda frames: [[t["tracking_id"] for t in fr["tracks"]] for fr in frames]    # noqa: E731
    assert ids(_restatement(greedy, "hungarian")) != ids(gold["frames"])


def test_default_opt_tracker_options_match_reference():
    ref = json.load(open(os.path.join(GOLDEN, "tracker_opt_defaults.json")))
    assert set(ref) == set(mgt.OPT_DEFAULT_FIELDS)
    for arch, trk in (("dla_34", False), ("dla_34", True), ("dlav1_34", False)):
        o = cpb.default_opt(arch, tracking_task=trk)
        for k, v in ref.items():
            assert getattr(o, k) == v, k
