"""Builds the reference's own CPU command line, oracle/_ref/racon_cpu (TEST INFRASTRUCTURE, recipe in oracle/refcli.mk):
what tests/golden/make_cli_cases.py runs to make the answers of tests/golden/cli_cases.json."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def build_refcli():
    """Keeps what is there when the reference sources are absent; returns the binary's path, or None without one."""
    out = os.path.join(HERE, "_ref", "racon_cpu")
    r = subprocess.run(["make", "-C", HERE, "-f", "Makefile", "-f", "refcli.mk", "refcli"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed (refcli):\n%s" % r.stdout)
    return out if os.path.exists(out) else None
