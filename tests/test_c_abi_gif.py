"""include/b200_caesium_gif.h is part of the C ABI: it must compile as strict C99, its entry points must link, and the host
decoder hook must work from a plain C program (tests/c_abi_gif_check.c) without a device."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")


def test_gif_header_is_c99_and_every_symbol_links(L, tmp_path):
    exe = str(tmp_path / "c_abi_gif_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "c_abi_gif_check.c"),
           "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "gif c-abi ok" in r.stdout


def test_gif_check_covers_every_declared_function():
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_gif.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr)) - {"b200_status"}
    src = open(os.path.join(ROOT, "tests", "c_abi_gif_check.c")).read()
    missing = [f for f in sorted(declared) if "(fn)" + f not in src]
    assert not missing, missing
