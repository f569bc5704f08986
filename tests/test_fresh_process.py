"""The fresh-process runner of tests/common.py, without the GPU (init=None: the child never loads
the library): what reaches the child, and how a failing body is reported."""
import os

import pytest

from tests import common


def _fresh_expect_env(bb, port, expected):
    """expected: {variable: value, or None for unset}."""
    assert bb.__name__ == "blitzar_b200" and port.__name__ == "oracle.port"
    for name, value in expected.items():
        assert os.environ.get(name) == value, (name, os.environ.get(name))
    print("checked", sorted(expected))


def _fresh_fail(bb, port, message):
    assert False, message


def test_arguments_and_env_reach_the_child(monkeypatch):
    monkeypatch.setenv("BLITZAR_LOG_LEVEL", "info")
    r = common.run_fresh((_fresh_expect_env, {"BLITZAR_LOG_LEVEL": "debug", "FRESH_CASE": "7"}),
                         (_fresh_expect_env, {"FRESH_CASE": "7"}), init=None,
                         env={"BLITZAR_LOG_LEVEL": "debug", "FRESH_CASE": "7"})
    assert r.stdout.splitlines()[:2] == ["checked ['BLITZAR_LOG_LEVEL', 'FRESH_CASE']",
                                         "checked ['FRESH_CASE']"]


def test_library_variables_of_this_process_are_stripped(monkeypatch):
    monkeypatch.setenv("BLITZAR_B200_DEVICES", "2")
    monkeypatch.setenv("BLITZAR_PARTITION_WINDOW_WIDTH", "5")
    monkeypatch.setenv("FRESH_PARENT", "kept")
    common.run_fresh((_fresh_expect_env, {"BLITZAR_B200_DEVICES": None,
                                          "BLITZAR_PARTITION_WINDOW_WIDTH": None,
                                          "FRESH_PARENT": "kept"}), init=None)


def test_failing_body_raises_with_its_message():
    with pytest.raises(AssertionError, match="body 3 of the fresh case failed"):
        common.run_fresh((_fresh_fail, "body 3 of the fresh case failed"), init=None)
