"""Host-only checks of the plan-cache ABI: the ctypes mirror of i2it_memory_stats follows the header field for field, and the
new calls refuse a NULL handle (no GPU needed)."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CTYPES = {"size_t": C.c_size_t, "int": C.c_int}


def _header_fields(struct):
    hdr = open(os.path.join(ROOT, "include", "i2it.h")).read()
    body = re.search(rf"typedef struct {struct} \{{(.*?)\}} {struct};", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        ctype, names = decl.split(None, 1)
        fields += [(n.strip(), ctype) for n in names.split(",")]
    return fields


def test_memory_stats_mirror_matches_header():
    import i2it
    hdr = _header_fields("i2it_memory_stats")
    assert [n for n, _ in hdr] == ["arena_bytes", "plan_bytes", "plans", "plan_builds", "plan_evictions"]
    assert [(n, _CTYPES[t]) for n, t in hdr] == list(i2it.MemoryStats._fields_)


def test_plan_cache_calls_refuse_a_null_handle():
    import i2it
    lib = i2it.load_library()
    s = i2it.MemoryStats()
    assert lib.i2it_memory_stats_get(None, C.byref(s)) == 1
    assert lib.i2it_set_max_plans(None, 4) == 1
    assert lib.i2it_release_plans(None) == 1
    assert lib.i2it_debug_poison_workspace(None, 0xFF) == 1
