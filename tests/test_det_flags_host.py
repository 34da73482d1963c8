"""Host: --deterministic is an opt-in extension of main.py's flags.  Without it the parsed flag set is exactly the
parent's (the attribute is absent); with it the run selects the fixed-order reductions."""
from tests.test_train_monitoring_host import PARENT_FLAG_DEFAULTS


def test_deterministic_flag_is_opt_in():
    import main as M
    assert vars(M.parse_flags([])) == PARENT_FLAG_DEFAULTS
    assert not hasattr(M.parse_flags([]), "deterministic")
    assert M.parse_flags(["--deterministic"]).deterministic is True
    assert M.parse_flags(["--deterministic", "true"]).deterministic is True
    assert M.parse_flags(["--nodeterministic"]).deterministic is False
    assert vars(M.parse_flags(["--deterministic"])) == dict(PARENT_FLAG_DEFAULTS, deterministic=True)
    assert M.parse_flags(["--noflip"]).flip is False and M.parse_flags([]).flip is True
