"""capi.ABI, the one description of every library's C ABI that the loaders apply, against the headers under include/:
the same symbols, and for each one as many argtypes as the prototype has parameters."""
import re

from conftest import REPO
from cuda_l2_b200 import capi

# a prototype's name and parameter list: `<return type> b200_name(<params>);`, possibly over several lines
PROTO = re.compile(r"^[A-Za-z][\w\s\*]*?\b(b200_\w+)\s*\(([^()]*)\)\s*;", re.M)


def prototypes() -> dict[str, int]:
    """Every b200_* prototype of every header -> its parameter count ((void) counts as 0)."""
    out = {}
    for header in sorted((REPO / "include").glob("*.h")):
        text = re.sub(r"/\*.*?\*/|//[^\n]*", "", header.read_text(), flags=re.S)
        for name, params in PROTO.findall(text):
            params = " ".join(params.split())
            assert name not in out, f"{name} is declared twice"
            out[name] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def table() -> dict[str, tuple]:
    out = {}
    for lib, symbols in capi.ABI.items():
        for name, sig in symbols.items():
            assert name not in out, f"{name} is in the table twice"
            out[name] = sig
    return out


def test_headers_declare_the_known_prototypes():
    protos = prototypes()
    assert len(protos) == 57
    assert protos["b200_hgemm_num_configs"] == 0 and protos["b200_hgemm_schedule_units"] == 13


def test_every_prototype_is_in_the_table_and_nothing_else():
    assert sorted(table()) == sorted(prototypes())


def test_argtypes_match_the_parameter_counts():
    protos = prototypes()
    wrong = {name: (len(args), protos[name]) for name, (args, _) in table().items() if len(args) != protos[name]}
    assert not wrong, f"argtypes length != parameter count: {wrong}"

