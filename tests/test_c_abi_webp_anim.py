"""include/b200_caesium_webp_anim.h is part of the C ABI: it must compile as strict C99, its entry points must link, and the host
decoder hook must work from a plain C program (tests/c_abi_webp_anim_check.c) without a device."""
import os
import re
import subprocess

import webp_anim_cases as wc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")


def test_webp_anim_header_is_c99_and_every_symbol_links(L, tmp_path):
    exe = str(tmp_path / "c_abi_webp_anim_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_webp_anim_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    src = tmp_path / "odd_1x1.webp"
    src.write_bytes(wc.hand_cases()["odd_1x1"])
    r = subprocess.run([exe, str(src)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "webp anim c-abi ok" in r.stdout


def test_webp_anim_check_covers_every_declared_function():
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_webp_anim.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr)) - {"b200_status"}
    src = open(os.path.join(ROOT, "tests", "c_abi_webp_anim_check.c")).read()
    missing = [f for f in sorted(declared) if "(fn)" + f not in src]
    assert not missing, missing
