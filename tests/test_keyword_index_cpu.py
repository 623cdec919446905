"""The term-major index's C entry points without a GPU: refusals before any device work, and the header's
aur_kw_index_stats layout equal to the binding's."""

import ctypes as C
import os
import re

from aurora_b200 import _native as N


def test_index_entry_points_refuse_bad_arguments():
    from aurora_b200.build import build_native

    build_native()
    lib = N.load()
    assert lib.aur_kw_reindex(None) == N.AUR_ERR_INVALID
    assert lib.aur_kw_set_option(None, b"kw_path", 1) == N.AUR_ERR_INVALID
    assert lib.aur_kw_get_index_stats(None, None) == N.AUR_ERR_INVALID
    st = N.AurKwIndexStats()
    assert lib.aur_kw_get_index_stats(None, C.byref(st)) == N.AUR_ERR_INVALID
    assert b"null" in lib.aur_last_error()


def test_header_declares_the_index_stats_layout_and_exports():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "aurora_b200.h")).read()
    flat = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    body = re.search(r"typedef struct aur_kw_index_stats \{(.*?)\} aur_kw_index_stats;", flat, re.S).group(1)
    names = [n.strip() for decl in body.split(";") if decl.strip() for n in decl.split(None, 1)[1].split(",")]
    assert names == [f for f, _ in N.AurKwIndexStats._fields_]
    assert C.sizeof(N.AurKwIndexStats) == 48
    assert int(re.search(r"#define AUR_KW_PATH_FORWARD (\d+)", hdr).group(1)) == N.KW_PATH_FORWARD
    assert int(re.search(r"#define AUR_KW_PATH_INDEX (\d+)", hdr).group(1)) == N.KW_PATH_INDEX
    for name in ("aur_kw_reindex", "aur_kw_set_option", "aur_kw_get_index_stats"):
        assert re.search(rf"\bint {name}\(", flat) and name in N.EXPORTS
