"""Deterministic training's host side: the commands' -deterministic option and vd_set_deterministic's refusal of a null
engine (the binding itself is checked against the header by test_abi.py)."""
import pytest

from visdial_b200 import _lib, cli


@pytest.mark.parametrize("argv,want", [([], 0), (["-deterministic", "1"], 1), (["-deterministic", "0"], 0)])
def test_deterministic_parses(argv, want):
    for options in (cli.TRAIN_OPTIONS, cli.FINETUNE_OPTIONS, cli.EVALUATE_OPTIONS, cli.GENERATE_COMMAND_OPTIONS):
        assert cli.parse(options, argv, prog="t").get("deterministic", 0) == want


@pytest.mark.parametrize("argv", [["-deterministic", "2"], ["-deterministic", "-1"], ["-deterministic", "yes"],
                                  ["-deterministic"], ["-deterministic", "1", "-gpus", "2"]])
def test_deterministic_rejects_other_values(argv, capsys):
    with pytest.raises(SystemExit) as e:
        cli.parse(cli.TRAIN_OPTIONS, argv, prog="t")
    assert e.value.code == 2 and "-deterministic" in capsys.readouterr().err


def test_deterministic_is_not_a_model_parameter():
    opt = cli.parse(cli.TRAIN_OPTIONS, ["-deterministic", "1"], prog="t")
    assert "deterministic" not in cli.model_params(opt)


def test_set_deterministic_refuses_a_null_engine():
    lib = _lib.load()
    assert lib.vd_set_deterministic(None, 1) == -1
    assert lib.vd_set_deterministic(None, 0) == -1
