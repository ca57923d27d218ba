"""CPU: the library's text vocabulary parser (sivo_dbg_vocabulary_parse, no device) against oracle/bow_oracle.py's parser, array for
array, on written trees, and SIVO_EFORMAT for each damaged form."""
import numpy as np
import pytest

from oracle import bow_oracle as B
from oracle import bow_scene as S
from sivo_b200 import _lib as L
from sivo_b200.bow import parse_text


def _write(tmp_path, name, text):
    p = tmp_path / name
    p.write_bytes(text.encode())
    return str(p)


def _same(got, want):
    for k in ("k", "L", "scoring", "weighting"):
        assert got[k] == want[k]
    for k in ("parent", "is_leaf", "desc"):
        np.testing.assert_array_equal(got[k], want[k])
    np.testing.assert_array_equal(got["weight"].view(np.uint64), want["weight"].view(np.uint64))


@pytest.mark.parametrize("kind,seed", [("small", 0), ("small", 1), ("irregular", 2), ("irregular", 3)])
@pytest.mark.parametrize("tail", ["\n", "\n\n", "", "\n  \n\t\n"])
def test_library_parser_equals_the_oracle(tmp_path, kind, seed, tail):
    tree = S.small_tree(seed, scoring=seed % 6, weighting=seed % 4) if kind == "small" else S.irregular_tree(seed)
    text = B.to_text(tree, trailing=tail)
    got = parse_text(_write(tmp_path, "voc.txt", text))
    want = B.parse_text(text)
    _same(got, want)
    _same(got, tree)


def test_descriptor_bytes_wrap_and_weights_round_trip(tmp_path):
    text = "3 2 0 0\n0 1 " + " ".join(["300", "-1", "+7"] + ["0"] * 29) + " 0.1000000000000000055511151231257827 trailing tokens\n"
    got = parse_text(_write(tmp_path, "v.txt", text))
    want = B.parse_text(text)
    _same(got, want)
    assert list(got["desc"][1][:3]) == [44, 255, 7] and got["weight"][1] == 0.1


def _damaged(tree):
    lines = B.to_text(tree, trailing="").split("\n")
    node = lines[3].split()
    cases = {
        "k": ["21 6 0 0"] + lines[1:], "k_neg": ["-1 6 0 0"] + lines[1:], "L0": ["10 0 0 0"] + lines[1:], "L11": ["10 11 0 0"] + lines[1:],
        "scoring": ["10 6 6 0"] + lines[1:], "weighting": ["10 6 0 4"] + lines[1:], "header_short": ["10 6 0"] + lines[1:],
        "parent_ahead": lines[:3] + [" ".join(["99999"] + node[1:])] + lines[4:],
        "parent_self": lines[:3] + [" ".join(["3"] + node[1:])] + lines[4:],
        "parent_neg": lines[:3] + [" ".join(["-1"] + node[1:])] + lines[4:],
        "short_line": lines[:3] + [" ".join(node[:30])] + lines[4:],
        "no_weight": lines[:3] + [" ".join(node[:34])] + lines[4:],
        "bad_token": lines[:3] + [" ".join(node[:5] + ["x"] + node[6:])] + lines[4:],
        "blank_mid": lines[:4] + [""] + lines[4:],
        "truncated_last": lines[:-1] + [" ".join(lines[-1].split()[:20])],
        "empty_tree": lines[:1],
        "empty_file": [],
    }
    leaf_ids = [i for i in range(1, len(tree["parent"])) if tree["is_leaf"][i]]
    cases["leaf_parent"] = lines + [" ".join([str(leaf_ids[0]), "1"] + ["0"] * 32 + ["1.0"])]
    cases["childless_nonleaf"] = lines + [" ".join(["0", "0"] + ["1"] * 32 + ["0.5"])]  # a non-leaf child of the root, last
    return {k: "\n".join(v) + ("\n" if v else "") for k, v in cases.items()}


@pytest.mark.parametrize("case", ["k", "k_neg", "L0", "L11", "scoring", "weighting", "header_short", "parent_ahead", "parent_self",
                                  "parent_neg", "short_line", "no_weight", "bad_token", "blank_mid", "truncated_last", "empty_tree",
                                  "empty_file", "leaf_parent", "childless_nonleaf"])
def test_damaged_files_are_refused(tmp_path, case):
    text = _damaged(S.small_tree(5))[case]
    with pytest.raises(B.FormatError):
        B.parse_text(text)
    with pytest.raises(L.SivoError) as e:
        parse_text(_write(tmp_path, "bad.txt", text))
    assert e.value.code == L.EFORMAT


def test_missing_file_is_enoent(tmp_path):
    with pytest.raises(L.SivoError) as e:
        parse_text(str(tmp_path / "nope.txt"))
    assert e.value.code == L.ENOENT
