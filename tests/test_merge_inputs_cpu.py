"""sam.MergeInputs (elprep_b200/sam.py) and elprep::MergeInputs (include/elprep_b200.hpp), the restatement of sam.MergeInputs
(sam/merge-inputs.go:16-219), against hand-worked cases from the reference code, and against each other.  No GPU."""
import os
import random
import subprocess

import pytest

from elprep_b200 import sam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def H(sq=(), rg=(), pg=()):
    h = sam.Header(sq=[{"SN": s, "LN": 100 + i} for i, s in enumerate(sq)],
                   rg=[dict(r) if isinstance(r, dict) else {"ID": r} for r in rg])
    h.PG = [{"ID": p} for p in pg]
    return h


def names(h):
    return [s["SN"] for s in h.SQ]


def test_dictionaries_interleaved_and_appended():
    m, maps, rg, pg = sam.MergeInputs([H(["c1", "c3"]), H(["c1", "c2", "c3"])], "S")
    assert names(m) == ["c1", "c2", "c3"] and maps == [[0, 2], [0, 1, 2]] and rg == {} and pg == {}
    m, maps, _, _ = sam.MergeInputs([H(["c1"]), H(["c2"]), H(["c0", "c1"])], "S")
    assert names(m) == ["c0", "c1", "c2"] and maps == [[1], [2], [0, 1]]
    assert m.HDSO() == sam.Unknown


def test_dictionary_conflict_panics():
    with pytest.raises(ValueError, match=r"^Cannot merge sequence dictionaries\.$"):
        sam.MergeInputs([H(["c1", "c2"]), H(["c2", "c1"])], "S")


def test_dictionary_index_quirks():
    # a shared entry sets j from its index in the new dictionary: from[j:] appends A a second time
    m, maps, _, _ = sam.MergeInputs([H(["A", "Z"]), H(["P", "Z", "A"])], "S")
    assert names(m) == ["P", "Z", "A", "A"] and maps == [[2, 1], [0, 1, 2]]
    # ... and a later from[j:iFrom] with j > iFrom is Go's slice panic
    with pytest.raises(ValueError, match=r"slice bounds out of range \[4:3\]"):
        sam.MergeInputs([H(["X", "Y", "A", "Z", "Q"]), H(["P", "Z", "A", "Q"])], "S")


def test_read_groups_three_files():
    m, _, rg, pg = sam.MergeInputs([H(rg=["1", "2"]), H(rg=["1", "1S"]), H(rg=["1S", "2"])], "S")
    # file 2: "1" collides with the IDs before it; its "1S" does not, so the same new ID is there twice
    assert [r["ID"] for r in m.RG] == ["1", "2", "1S", "1S", "1SS", "2S"]
    # every read of every file runs 1->1S, 1S->1SS, 2->2S in that order
    assert rg == {"1": "1SS", "1S": "1SS", "2": "2S"} and pg == {}
    m, _, rg, _ = sam.MergeInputs([H(rg=["1"]), H(rg=["1"]), H(rg=["1"])], "S")
    assert [r["ID"] for r in m.RG] == ["1", "1S", "1S"] and rg == {"1": "1S"}


def test_program_lines_and_pp_quirk():
    f1 = H(rg=[{"ID": "r1"}, {"ID": "r2", "PP": "p1"}], pg=["p1", "p2"])
    f2 = H(rg=[{"ID": "r3", "PP": "p1"}, {"ID": "r4", "PP": "p1"}], pg=["p1"])
    m, _, rg, pg = sam.MergeInputs([f1, f2], "7")
    assert [r["ID"] for r in m.PG] == ["p1", "p2", "p17"] and pg == {"p1": "p17"} and rg == {}
    # the PP loop runs i over 1..len(file 2's RG)-1 but indexes the merged RG: r2 of file 1 changes, r3 and r4 do not
    assert [r.get("PP") for r in m.RG] == [None, "p17", "p1", "p1"]
    assert [r.get("PP") for r in f1.RG] == [None, "p1"]            # the inputs are not changed


def test_metadata_comments_user_records():
    a, b = H(["c"]), H(["c"])
    a.HD = {"VN": "1.5", "SO": "coordinate", "GO": "none"}
    b.HD = {"VN": "1.6"}
    a.CO, b.CO = ["x"], ["y"]
    a.UserRecords, b.UserRecords = {"@zz": [{"k": "1"}], "@aa": []}, {"@zz": [{"k": "2"}]}
    m = sam.MergeInputs([a, b], "S")[0]
    assert m.HD == {"VN": "1.6", "SO": "unknown", "GO": "none"} and m.CO == ["x", "y"]
    assert m.UserRecords == {"@zz": [{"k": "2"}], "@aa": []}
    assert sam.MergeInputs([a], "S")[0].HD["SO"] == "coordinate"   # one input: nothing merged


def _hx(s):
    return s.encode().hex()


def _encode(case):
    suffix, hs = case
    fields = [_hx(suffix)]
    for h in hs:
        sq = ",".join(_hx(s["SN"]) for s in h.SQ)
        rg = ",".join(_hx(r["ID"]) + ":" + (_hx(r["PP"]) if "PP" in r else "-") for r in h.RG)
        pg = ",".join(_hx(p["ID"]) for p in h.PG)
        fields.append(f"{sq};{rg};{pg}")
    return "\t".join(fields)


def _python_line(case):
    try:
        m, maps, rg, pg = sam.MergeInputs(case[1], case[0])
    except ValueError as e:
        return "PANIC " + _hx(str(e))
    mp = lambda d: ",".join(_hx(k) + ":" + _hx(d[k]) for k in sorted(d, key=lambda s: s.encode()))
    return "\t".join([",".join(_hx(s["SN"]) for s in m.SQ),
                      ",".join(_hx(r["ID"]) + ":" + (_hx(r["PP"]) if "PP" in r else "-") for r in m.RG),
                      ",".join(_hx(p["ID"]) for p in m.PG),
                      "|".join(",".join(str(i) for i in v) for v in maps), mp(rg), mp(pg)])


def test_cpp_equals_python(tmp_path):
    exe = str(tmp_path / "merge_inputs_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "merge_inputs_check.cpp"), "-o", exe])
    rnd = random.Random(5)
    pool = ["c1", "c2", "c3", "c4", "c5", "X"]
    cases = []
    for _ in range(3000):
        hs = []
        for _ in range(rnd.randint(1, 4)):
            sq = rnd.sample(pool, rnd.randint(0, 5))
            rg = [{"ID": rnd.choice(["1", "2", "1S", "2S", "1SS"])} for _ in range(rnd.randint(0, 3))]
            for r in rg:
                if rnd.random() < 0.4:
                    r["PP"] = rnd.choice(["p", "pS", "q"])
            hs.append(H(sq, rg, [rnd.choice(["p", "pS", "q"]) for _ in range(rnd.randint(0, 3))]))
            hs[-1].SQ = [{"SN": s, "LN": 1} for s in sq]
        cases.append(("S", hs))
    cases += [("S", [H(["X", "Y", "A", "Z", "Q"]), H(["P", "Z", "A", "Q"])]), ("S", [H(["A", "Z"]), H(["P", "Z", "A"])]),
              ("7", [H(rg=[{"ID": "r1"}, {"ID": "r2", "PP": "p1"}], pg=["p1", "p2"]), H(rg=[{"ID": "r3", "PP": "p1"}], pg=["p1"])])]
    out = subprocess.run([exe], input="\n".join(_encode(c) for c in cases) + "\n", capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    got = out.stdout.splitlines()
    assert len(got) == len(cases)
    kinds = set()
    for c, g in zip(cases, got):
        want = _python_line(c)
        assert g == want, (_encode(c), g, want)
        kinds.add(want.split(" ")[0] if want.startswith("PANIC") else "ok")
        if want.startswith("PANIC"):
            kinds.add(bytes.fromhex(want.split(" ")[1]).decode()[:13])
    assert {"ok", "PANIC", "Cannot merge ", "runtime error"} <= kinds
