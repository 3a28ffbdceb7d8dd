"""CPU: the streamed tile kernel's debug options (sb_debug_tile_options) are mirrored by saturn_b200/_lib.py."""
import os
import re

from saturn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tile_debug_option_names_match_the_library():
    """The TILE_DEBUG_* constants of _lib.py have the names and bits of the TileDebug enum in csrc/sb_internal.h, one
    distinct bit each, and sb_debug_tile_options / sb_debug_tile_wait are declared and bound."""
    src = open(os.path.join(ROOT, "saturn_b200", "csrc", "sb_internal.h")).read()
    enum = re.search(r"enum TileDebug : unsigned \{(.*?)\};", src, flags=re.S).group(1)
    in_c = {name: int(value) for name, value in re.findall(r"^\s*(TILE_DEBUG_\w+)\s*=\s*(\d+)u,", enum, flags=re.M)}
    in_py = {name: value for name, value in vars(_lib).items() if name.startswith("TILE_DEBUG_")}
    assert in_c == in_py and set(in_c) == {"TILE_DEBUG_TIMING", "TILE_DEBUG_ROW_COPIES", "TILE_DEBUG_NO_STAGGER"}
    assert all(bin(v).count("1") == 1 for v in in_py.values()) and len(set(in_py.values())) == len(in_py)
    with open(os.path.join(ROOT, "include", "saturn_b200.h")) as f:
        header = f.read()
    for sym in ("sb_debug_tile_options", "sb_debug_tile_wait"):
        assert sym in _lib.SYMBOLS and re.search(r"int\s+%s\s*\(" % sym, header)
