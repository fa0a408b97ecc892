"""mortal_b200/_cdecl.py: ctypes bindings and constants read from C declarations (CPU only)."""
import ctypes as C

import pytest

from mortal_b200 import _cdecl

SRC = r'''
#include <stdint.h>
typedef struct mjx_env mjx_env;
int mjx_outside(int x) { return x; }            /* a definition outside extern "C": not an entry */
extern "C" {
struct mjx_pair { int a, b; };
static int mjx_helper(float f) { return 0; }    // static: not exported
const char* mjx_name(void);
int mjx_create(mjx_env** out, long long n,
               const uint64_t* keys /* host */,
               double scale, void* stream);
uint8_t* mjx_view(mjx_env* env) { const char* s = "}{"; return (uint8_t*)s; }
void mjx_none();
int mjx_unnamed(long long, const int, uint8_t*);
int64_t mjx_wide(uint32_t a, int32_t b, int64_t c, uint64_t d, long e, float f, char* out, struct mjx_pair* p);
}
'''


def test_functions_read_prototypes_and_definitions():
    d = _cdecl.functions(SRC, "mjx_")
    assert set(d) == {"mjx_name", "mjx_create", "mjx_view", "mjx_none", "mjx_unnamed", "mjx_wide"}
    assert d["mjx_name"] == (C.c_char_p, [])
    assert d["mjx_none"] == (None, [])
    assert d["mjx_create"] == (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_double, C.c_void_p])
    assert d["mjx_view"] == (C.c_void_p, [C.c_void_p])
    assert d["mjx_unnamed"] == (C.c_int, [C.c_longlong, C.c_int, C.c_void_p])
    assert d["mjx_wide"] == (C.c_int64, [C.c_uint32, C.c_int32, C.c_int64, C.c_uint64, C.c_long, C.c_float, C.c_void_p,
                                          C.c_void_p])
    assert _cdecl.functions(SRC, "mjx_cr") == {"mjx_create": d["mjx_create"]}


@pytest.mark.parametrize("decl", ["int mjx_f(size_t n);", "unsigned mjx_f(int n);", "int mjx_f(void x);", "int mjx_f(int a[4]);",
                                  "bool mjx_f(void);"])
def test_functions_reject_unknown_types(decl):
    with pytest.raises(ValueError, match="mjx_f"):
        _cdecl.functions('extern "C" {\n' + decl + "\n}", "mjx_")


def test_bind_sets_types_and_fails_on_a_missing_export():
    libc = C.CDLL(None)
    _cdecl.bind(libc, {"strlen": (C.c_long, [C.c_char_p])})
    assert libc.strlen.restype is C.c_long and libc.strlen.argtypes == [C.c_char_p] and libc.strlen(b"abc") == 3
    with pytest.raises(AttributeError):
        _cdecl.bind(libc, {"mjx_not_exported_anywhere": (C.c_int, [])})


def test_constants():
    text = "#define A 7 /* c */\n#define B(x) x\n#define C -0x10\nenum e { P, Q = 5, R,\n S };\n" \
           '#define L(X) X(ONE, "one, 1") \\\n    X(TWO, "two")\n'
    assert _cdecl.defines(text) == {"A": 7, "C": -16}
    assert _cdecl.enum(text, "e") == {"P": 0, "Q": 5, "R": 6, "S": 7}
    assert _cdecl.xmacro(text, "L") == [("ONE", "one, 1"), ("TWO", "two")]
    with pytest.raises(ValueError):
        _cdecl.enum("enum f { A = B + 1 };", "f")


def test_header_constants_equal_their_python_names():
    from mortal_b200 import dataset, dataset_codec, stat, validate_logs

    import grp_lib

    assert validate_logs.STATUSES == ("OK", "CHECK", "UPDATE", "PARSE", "UNSUPPORTED")
    assert grp_lib.STATUS == {0: "OK", 1: "NO_DELTAS", 2: "NO_KYOKU", 3: "CAPACITY"}
    assert dataset_codec.HORA_WORDS == 2 and dataset._ERR_HIDDEN_OWN_TILE == 13
    assert len(validate_logs.REASONS) == 34 and validate_logs.REASONS[0] == "none" and validate_logs.REASONS[-1] == "capacity"
    assert validate_logs.REASONS[3] == "chi from non-kamicha"
    names = stat._read_counters()
    assert names[0] == "game" and names[-1] == "nagashi_mangan" and sorted(names) == sorted(stat.COUNTERS)
    assert _cdecl.enum(_cdecl.header(), "mjx_mw_event")["MJX_MW_T_END_KYOKU"] == 14
