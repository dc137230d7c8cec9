"""CPU test of the test-only library: every entry point defined in csrc/testing.cu is exported by libsdxl_b200_testing.so and
bound in sdxl_b200/_testing.py, and nothing else is, so a wrapper cannot be added without its binding or the reverse."""
import os
import re
import struct

from sdxl_b200 import _testing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def source_symbols():
    src = open(os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "csrc", "testing.cu")).read()
    return set(re.findall(r"SDXL_TEST_API\s+[\w\s\*]+?\b(sdxl_test_\w+)\s*\(", src))


def exported_symbols(path):
    """Names of the defined global / weak symbols in an ELF64 little-endian shared object's .dynsym."""
    data = open(path, "rb").read()
    assert data[:4] == b"\x7fELF" and data[4] == 2 and data[5] == 1, "expected an ELF64 little-endian object"
    shoff, = struct.unpack_from("<Q", data, 0x28)
    shentsize, shnum = struct.unpack_from("<HH", data, 0x3A)
    sections = [struct.unpack_from("<IIQQQQIIQQ", data, shoff + i * shentsize) for i in range(shnum)]
    names = set()
    for _, sh_type, _, _, off, size, link, _, _, entsize in sections:
        if sh_type != 11:                                   # SHT_DYNSYM
            continue
        stroff = sections[link][4]
        for i in range(size // entsize):
            st_name, st_info, _, st_shndx, _, _ = struct.unpack_from("<IBBHQQ", data, off + i * entsize)
            if st_shndx == 0 or (st_info >> 4) not in (1, 2):   # undefined, or neither STB_GLOBAL nor STB_WEAK
                continue
            end = data.index(b"\0", stroff + st_name)
            names.add(data[stroff + st_name:end].decode())
    return names


def test_testing_library_exports_match_bindings():
    if not os.path.exists(_testing.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    declared = source_symbols()
    assert len(declared) >= 50
    exported = {s for s in exported_symbols(_testing.LIB_PATH) if s.startswith("sdxl_test_")}
    assert declared == exported, f"testing.cu vs exports: only in source {declared - exported}, only exported {exported - declared}"
    assert declared == set(_testing.PROTOTYPES), \
        f"testing.cu vs PROTOTYPES: missing {declared - set(_testing.PROTOTYPES)}, extra {set(_testing.PROTOTYPES) - declared}"
    _testing.load()                                         # every prototype resolves
