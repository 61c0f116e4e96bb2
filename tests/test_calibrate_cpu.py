"""CPU: the host side of activation-range calibration: the exponent rule, the saved-ranges file, the C ABI declarations
and the command-line flag.  No GPU work."""
import json
import os
import re

import pytest

import ideepcolor_b200 as cli
from interactive_deep_colorization_b200 import _lib, engine, launcher
from tests import calibrate_ref, calibrated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rule_exact_powers_of_two():
    """max_abs = 2^k stores at exactly 2^kActExpCal: S = kActExpCal - k, not one less; just above 2^k takes one more."""
    for k in range(-20, 21):
        assert calibrate_ref.exponent_from_range(2.0 ** k) == calibrate_ref.ACT_EXP_CAL - k
        assert calibrate_ref.exponent_from_range(2.0 ** k * (1 + 2.0 ** -40)) == calibrate_ref.ACT_EXP_CAL - k - 1
        assert calibrate_ref.exponent_from_range(2.0 ** k * (1 - 2.0 ** -40)) == calibrate_ref.ACT_EXP_CAL - k
    for v in (0.3, 1.0, 77.0, 513.0, 4e5):
        stored = v * 2.0 ** calibrate_ref.exponent_from_range(v)
        assert 2.0 ** (calibrate_ref.ACT_EXP_CAL - 1) < stored <= 2.0 ** calibrate_ref.ACT_EXP_CAL


def test_precedence_and_partial_ranges(synth_sd):
    est = {b: e[2] for b, e in calibrated.act_estimates(synth_sd).items()}
    assert calibrate_ref.expected_exponents(synth_sd) == est
    ranges = {"conv4_3": 3000.0, "a8_1": 0.7, "a3_1": 0.0}            # a3_1 measured 0 (a dead layer): no range
    got = calibrate_ref.expected_exponents(synth_sd, ranges, overrides={"a8_1": 5})
    assert got["conv4_3"] == 10 - 12 and got["a8_1"] == 5 and got["a3_1"] == est["a3_1"]
    assert {b: s for b, s in got.items() if b not in ("conv4_3", "a8_1")} == \
        {b: s for b, s in est.items() if b not in ("conv4_3", "a8_1")}
    assert calibrate_ref.expected_exponents(synth_sd, ranges)["a8_1"] == 10 - 0


def test_stale_statistics_network_is_the_same_function_with_a_large_conv4_3(synth_sd):
    sd = calibrate_ref.stale_statistics(synth_sd)
    est0, est1 = calibrated.act_estimates(synth_sd), calibrated.act_estimates(sd)
    assert est1["conv4_3"][2] == est0["conv4_3"][2]                    # the statistics did not move: same estimate
    assert est1["a4_2"][2] == est0["a4_2"][2]


def test_json_round_trip(tmp_path):
    r = {"conv4_3": 3123.4567, "a8_1": 0.7, "hyper": 2.0 ** -9}
    p = str(tmp_path / "ranges.json")
    engine.save_act_ranges(p, r)
    assert engine.load_act_ranges(p) == r
    assert json.load(open(p)) == r                                     # a flat JSON object
    assert engine.resolve_calibration(p, None) == r and engine.resolve_calibration(r, None) == r
    assert engine.resolve_calibration(None, None) is None
    assert engine.resolve_calibration(["photo"], lambda photos: {"a1_1": float(len(photos))}) == {"a1_1": 1.0}


@pytest.mark.parametrize("entry,word", [({"conv4_3": float("nan")}, "conv4_3"), ({"conv4_3": float("inf")}, "conv4_3"),
                                        ({"a8_1": 0.0}, "a8_1"), ({"a8_1": -3.0}, "a8_1"), ({"a8_1": "7"}, "a8_1"),
                                        ({"a8_1": True}, "a8_1"), ({"conv99": 1.0}, "conv99"), ([1.0], "object")])
def test_bad_ranges_are_rejected_by_name(tmp_path, entry, word):
    with pytest.raises(ValueError, match=word):
        engine.check_act_ranges(entry)
    p = str(tmp_path / "bad.json")
    json.dump(entry, open(p, "w"))
    with pytest.raises(ValueError, match=word):
        engine.load_act_ranges(p)
    with pytest.raises(ValueError):
        engine.save_act_ranges(str(tmp_path / "never.json"), entry)
    assert not os.path.exists(str(tmp_path / "never.json")) or os.path.getsize(str(tmp_path / "never.json")) == 0


def test_buffer_list_matches_the_plan():
    assert sorted(engine.ACT_BUFFERS) == sorted(b for b, _, _ in calibrated._PLAN)


_C2CT = {"idc_ctx*": "c_void_p", "const char*": "c_char_p", "int": "c_int", "float*": "LP_c_float", "double": "c_double"}


def test_new_symbols_declared_alike_in_header_and_ctypes():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "idc_b200.h")).read(), flags=re.S)
    table = {n: (res, args) for n, res, args in _lib.SYMBOLS}
    for name in ("idc_num_acts", "idc_act_name", "idc_act_absmax", "idc_set_act_range"):
        m = re.search(r"(int|const char\*)\s+%s\s*\(([^)]*)\)\s*;" % name, src)
        assert m, name
        params = [re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*") for a in m.group(2).split(",")]
        res, args = table[name]
        assert res.__name__ == _C2CT[m.group(1)], name
        assert [a.__name__ for a in args] == [_C2CT[p] for p in params], (name, params)


def test_cli_calibrate_argument(tmp_path, capsys):
    d = tmp_path / "photos"
    d.mkdir()
    for i in range(20):
        (d / ("p%02d.png" % i)).write_bytes(b"")
    (d / "notes.txt").write_bytes(b"")
    j = tmp_path / "r.json"
    engine.save_act_ranges(str(j), {"conv4_3": 10.0})
    for parse, base in ((cli.parse_args, ["--color_model", "w.pth"]), (launcher.parse_args, [])):
        a = parse(base + ["--calibrate", str(d)])
        assert len(a.calibrate_source) == 16 and a.calibrate_source == sorted(a.calibrate_source)
        assert all(p.endswith(".png") and os.path.dirname(p) == str(d) for p in a.calibrate_source)
        assert parse(base + ["--calibrate", str(d)]).calibrate_source == a.calibrate_source       # seeded
        assert parse(base + ["--calibrate", str(j)]).calibrate_source == str(j)
        assert parse(base).calibrate_source is None
        with pytest.raises(SystemExit):
            parse(base + ["--calibrate", str(tmp_path / "missing")])
        assert "missing" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.parse_args(["--color_model", "w.pth", "--save_act_ranges", "x.json"])
    assert cli.parse_args(["--color_model", "w.pth", "--calibrate", str(j), "--save_act_ranges", "x.json"]).save_act_ranges == "x.json"
