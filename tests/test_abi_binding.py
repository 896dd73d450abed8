"""CPU (-m "not gpu"): the ctypes binding and the run-time options of the C ABI are read from include/latex_ocr_b200.h.  Every
function's argtypes / restype equal the parse of its prototype (spot-checked against signatures written out here); the library's
option table holds exactly the options the header documents, with their documented defaults; _lib.option restores."""
import ctypes
import json
import os
import re
import subprocess
import sys

import pytest

from latex_ocr_b200 import _lib

vp, i32, i64, f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float


def test_every_declared_function_is_bound_as_the_header_declares_it():
    L = _lib.lib()
    sigs = _lib.declared_signatures()
    assert sorted(sigs) == _lib.declared_symbols()
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(L, name)
        assert fn.restype == restype and list(fn.argtypes) == argtypes, name


@pytest.mark.parametrize("name,restype,argtypes", [
    ("lo_gemm", i32, [vp, i32, vp, i32, vp, i32, i32, i32, i32, i64, i64, i64, i64, i64, i32, i64, i64, i64, vp, i32, i32, i32, vp]),
    ("lo_tf_optim_step", i32, [i32] + [vp] * 5 + [i64, vp] + [f32] * 4 + [vp]),
    ("lo_attention_step_backward", i32, [vp] * 2 + [i32] + [vp] * 20 + [i32] * 6 + [vp, vp]),
    ("lo_get_option", i32, [ctypes.c_char_p]),
    ("lo_option_name", ctypes.c_char_p, [i32]),
    ("lo_attention_workspace_bytes", i64, [i32, i32]),
    ("lo_decoder_forward", i32, [ctypes.POINTER(_lib.DecoderArgs), i32, vp]),
])
def test_parsed_signatures_spot_checks(name, restype, argtypes):
    got_restype, got_argtypes = _lib.declared_signatures()[name]
    assert got_restype == restype and got_argtypes == argtypes
    if name == "lo_gemm":
        assert len(got_argtypes) == 23
        assert [i for i, t in enumerate(got_argtypes) if t == i64] == [9, 10, 11, 12, 13, 15, 16, 17]


def _documented_options():
    """{name: default} of the option list in the header's comment above lo_set_option."""
    with open(_lib.HEADER) as f:
        text = f.read()
    block = text[text.index("Run-time options."):text.index("int lo_set_option(")]
    return {name: int(default) for name, default in re.findall(r"^ \*   (\w+) +(-?\d+)\b", block, re.M)}


# runs in a fresh interpreter without LO_OPTS, so that every option still holds its default
_PROBE = r"""
import json
from latex_ocr_b200 import _lib
L = _lib.lib()
get = lambda n: L.lo_get_option(n.encode())
names = []
while L.lo_option_name(len(names)) is not None:
    names.append(L.lo_option_name(len(names)).decode())
out = {"names": names, "defaults": {n: get(n) for n in names}, "roundtrip": {}}
for n in names:
    if n == "l2_persist_mb":             # an action on the device, not only a stored value
        continue
    for v in (7, -3, 0, 123456):
        out["roundtrip"].setdefault(n, []).append([L.lo_set_option(n.encode(), v), get(n)])
    L.lo_set_option(n.encode(), out["defaults"][n])
out["unknown"] = {}
for n in ("no_such_option", "fuse_lstm", "dec_streams", "conv_persist", "conv_mt2"):
    rc = L.lo_set_option(n.encode(), 1)
    out["unknown"][n] = [rc, L.lo_last_error().decode(), get(n)]
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def probe():
    root = os.path.dirname(os.path.dirname(_lib.HEADER))
    env = {k: v for k, v in os.environ.items() if k != "LO_OPTS"}
    env["PYTHONPATH"] = os.pathsep.join([root] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-s", "-c", _PROBE], cwd=root, env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_the_library_has_exactly_the_documented_options(probe):
    documented = _documented_options()
    assert len(documented) >= 16
    assert probe["names"] == list(documented)
    assert probe["defaults"] == documented


def test_every_stored_option_reads_back_what_was_set(probe):
    assert sorted(probe["roundtrip"]) == sorted(set(probe["names"]) - {"l2_persist_mb"})
    for name, pairs in probe["roundtrip"].items():
        assert pairs == [[0, 7], [0, -3], [0, 0], [0, 123456]], name


def test_unknown_option_is_refused(probe):
    # fuse_lstm, dec_streams, conv_persist and conv_mt2 were options until their schedules were removed: an LO_OPTS that still
    # names one fails on load
    assert sorted(probe["unknown"]) == ["conv_mt2", "conv_persist", "dec_streams", "fuse_lstm", "no_such_option"]
    for name, (rc, err, got) in probe["unknown"].items():
        assert rc == -1, name                                          # LO_EINVAL
        assert name in err
        assert got == -1, name


def test_option_restores_previous_values():
    L = _lib.lib()

    def get(*names):
        return [L.lo_get_option(n.encode()) for n in names]

    before = get("att_nsplit", "dbg_skip")
    with _lib.option(att_nsplit=5):
        with _lib.option(att_nsplit=9, dbg_skip=3):
            assert get("att_nsplit", "dbg_skip") == [9, 3]
        assert get("att_nsplit", "dbg_skip") == [5, before[1]]       # back to 5, not to the default
        with pytest.raises(ZeroDivisionError):
            with _lib.option(att_nsplit=7, dbg_skip=1):
                assert get("att_nsplit", "dbg_skip") == [7, 1]
                1 / 0
        assert get("att_nsplit", "dbg_skip") == [5, before[1]]
        with pytest.raises(_lib.LatexOcrB200Error, match="no_such_option"):
            with _lib.option(dbg_skip=2, no_such_option=1):
                pass
        assert get("att_nsplit", "dbg_skip") == [5, before[1]]
    assert get("att_nsplit", "dbg_skip") == before
