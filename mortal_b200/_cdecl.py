"""ctypes bindings and integer constants read from C declarations, so that include/mjx.h (and the test libraries' extern "C"
blocks) stay the only copy of every signature and mirrored value.

    functions(text, prefix)  {name: (restype, argtypes)} of the functions named prefix* in the extern "C" blocks of `text`
    bind(lib, decls)         set restype / argtypes on every declared entry of a loaded library
    defines(text)            {NAME: value} of every `#define NAME <integer>`
    enum(text, name)         {MEMBER: value} of `enum name { ... }`, in declaration order
    xmacro(text, name)       the argument tuples of the X(...) entries of `#define name(X) ...`
    header()                 the text of include/mjx.h
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mjx.h")

# The closed type map: a pointer is c_void_p (c_char_p for `const char*`), a scalar must be listed here, anything else raises.
_SCALARS = {"void": None, "int": C.c_int, "long": C.c_long, "long long": C.c_longlong, "int32_t": C.c_int32,
            "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float, "double": C.c_double}
# a parameter whose last word is one of these is unnamed (`long long`, `const int`): that word is part of its type
_TYPE_WORDS = {"void", "char", "int", "long", "short", "signed", "unsigned", "float", "double", "const"}
_LEXEMES = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
_DIRECTIVE = re.compile(r"^[ \t]*#(?:[^\n]*\\\n)*[^\n]*", re.M)
_INT = r"-?(?:0[xX][0-9a-fA-F]+|\d+)"


@functools.lru_cache(maxsize=None)
def header() -> str:
    with open(HEADER) as f:
        return f.read()


def _uncomment(text: str, keep_strings: bool = True) -> str:
    """`text` with comments blanked; keep_strings=False also empties string and character literals (all but `"C"`)"""
    def sub(m):
        s = m.group()
        if s[0] == "/":
            return "\n" * s.count("\n") or " "
        return s if keep_strings or s == '"C"' else s[0] * 2
    return _LEXEMES.sub(sub, text)


def _ctype(decl: str, text: str, result: bool):
    tokens = re.findall(r"\w+|\*", text)
    if "*" in tokens:
        return C.c_char_p if tokens == ["const", "char", "*"] else C.c_void_p
    key = " ".join(t for t in tokens if t != "const")
    if key not in _SCALARS or (key == "void" and not result):
        raise ValueError(f"cannot bind {key or text!r} in `{decl}`")
    return _SCALARS[key]


def _top_level(body: str):
    """the statements at brace depth 0 of `body`, each cut at its `;` or at the `{` of its block (blocks are skipped)"""
    stmts, start, depth = [], 0, 0
    for i, ch in enumerate(body):
        if ch == "{":
            if depth == 0:
                stmts.append(body[start:i])
            depth += 1
        elif ch == "}":
            depth -= 1
            if depth == 0:
                start = i + 1
        elif ch == ";" and depth == 0:
            stmts.append(body[start:i])
            start = i + 1
    return stmts


def _extern_c_blocks(text: str):
    for m in re.finditer(r'\bextern\s*"C"\s*\{', text):
        depth = 1
        for i in range(m.end(), len(text)):
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            if depth == 0:
                yield text[m.end():i]
                break


def functions(text: str, prefix: str) -> dict:
    """{name: (restype, argtypes)} of every function whose name starts with `prefix`, declared (`...;`) or defined (`...{`) inside
    an extern "C" block of the C / C++ source `text`; static functions are skipped. A type outside the closed map raises
    ValueError."""
    text = _DIRECTIVE.sub("", _uncomment(text, keep_strings=False))
    out = {}
    for block in _extern_c_blocks(text):
        for stmt in _top_level(block):
            stmt = " ".join(stmt.split())
            m = re.fullmatch(r"(\w[\w\s*]*?)\s*\b(" + re.escape(prefix) + r"\w*)\s*\((.*)\)", stmt)
            if not m or m[1].split()[0] in ("static", "typedef"):
                continue
            ret, name, params = m.groups()
            argtypes = []
            if params.strip() not in ("", "void"):
                for p in params.split(","):
                    p = p.strip()
                    named = re.fullmatch(r"(.*[\s*])(\w+)", p)
                    argtypes.append(_ctype(stmt, named[1] if named and named[2] not in _TYPE_WORDS else p, False))
            out[name] = (_ctype(stmt, ret, True), argtypes)
    return out


def bind(lib, decls: dict):
    """Set restype and argtypes of every entry of `decls` on `lib`; AttributeError if the library does not export one."""
    for name, (restype, argtypes) in decls.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


def defines(text: str) -> dict:
    return {name: int(v, 0) for name, v in
            re.findall(r"^[ \t]*#[ \t]*define[ \t]+(\w+)[ \t]+(" + _INT + r")[uUlL]*[ \t]*$", _uncomment(text), re.M)}


def enum(text: str, name: str) -> dict:
    """the members of `enum name`: an explicit integer value, or the previous member's value + 1 (0 for the first)"""
    m = re.search(r"\benum\s+" + re.escape(name) + r"\s*\{([^}]*)\}", _uncomment(text))
    if m is None:
        raise ValueError(f"no enum {name}")
    out, value = {}, -1
    for member in filter(None, (s.strip() for s in m[1].split(","))):
        e = re.fullmatch(r"(\w+)(?:\s*=\s*(" + _INT + r"))?", member)
        if e is None:
            raise ValueError(f"cannot read enum {name} member {member!r}")
        value = int(e[2], 0) if e[2] else value + 1
        out[e[1]] = value
    return out


def xmacro(text: str, name: str) -> list:
    """the arguments of every X(...) in `#define name(X) ...`, one tuple per entry; string literals are returned unquoted"""
    m = re.search(r"^[ \t]*#[ \t]*define[ \t]+" + re.escape(name) + r"\((\w+)\)((?:[^\n]*\\\n)*[^\n]*)", _uncomment(text), re.M)
    if m is None:
        raise ValueError(f"no X-macro {name}")
    lit = r'"(?:\\.|[^"\\])*"'
    entries = re.findall(r"\b" + m[1] + r"\(((?:" + lit + r'|[^()"])*)\)', m[2])
    return [tuple(a[1:-1] if a.startswith('"') else a for a in (s.strip() for s in re.findall(lit + r'|[^,"]+', e)) if a)
            for e in entries]
