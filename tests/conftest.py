import gzip, os, subprocess, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE); sys.path.insert(0, ROOT)
GOLD = os.path.join(HERE, "golden")

GOLDEN_CONFIGS = {
    "mem_default": dict(mode="mem"), "mem_noseg": dict(mode="mem", seg=False), "mem_m5": dict(mode="mem", m=5),
    "greedy_default": dict(mode="greedy"), "greedy_e5": dict(mode="greedy", e=5), "greedy_e1_s40": dict(mode="greedy", e=1, s=40),
    "greedy_e0": dict(mode="greedy", e=0), "greedy_noseg": dict(mode="greedy", seg=False),
}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    # a GPU test that hangs (a deadlocked pipeline, a kernel that never ends) must not hold the box: ten minutes per test (pytest-timeout)
    if config.pluginmanager.hasplugin("timeout"):
        for it in items:
            if it.get_closest_marker("gpu") and not it.get_closest_marker("timeout"):
                it.add_marker(pytest.mark.timeout(600))


def _read_fq_gz(path):
    names, seqs = [], []
    with gzip.open(path, "rt") as f:
        lines = f.read().split("\n")
    for i in range(0, len(lines) - 3, 4):
        name = lines[i][1:]
        for k, ch in enumerate(name):
            if ch in " /\t\r":
                name = name[:k]; break
        names.append(name); seqs.append("".join(c for c in lines[i + 1] if c.isalpha()))
    off = np.zeros(len(seqs) + 1, dtype=np.uint64); off[1:] = np.cumsum([len(s) for s in seqs])
    return names, np.frombuffer("".join(seqs).encode(), dtype=np.uint8).copy(), off


class Golden:
    fmi = os.path.join(GOLD, "db.fmi"); nodes = os.path.join(GOLD, "nodes.dmp")

    def __init__(self):
        self.pe = (_read_fq_gz(os.path.join(GOLD, "pe150_1.fq.gz")), _read_fq_gz(os.path.join(GOLD, "pe150_2.fq.gz")))
        self.se = _read_fq_gz(os.path.join(GOLD, "se100.fq.gz"))

    def reads(self, tag):
        if tag == "pe150":
            (n1, s1, o1), (n2, s2, o2) = self.pe
            assert n1 == n2
            return n1, s1, o1, s2, o2
        n, s, o = self.se
        return n, s, o, None, None

    def expected(self, cfg, tag):
        tax, best, ids = [], [], []
        with gzip.open(os.path.join(GOLD, "expected_%s_%s.tsv.gz" % (cfg, tag)), "rt") as f:
            for line in f:
                p = line.rstrip("\n").split("\t")
                tax.append(int(p[2])); best.append(int(p[3])); ids.append(tuple(int(x) for x in p[4].split(",") if x))
        return np.array(tax, dtype=np.uint64), np.array(best, dtype=np.uint32), ids


@pytest.fixture(scope="session")
def golden():
    return Golden()


@pytest.fixture(scope="session")
def built():
    """Make sure the oracle, the generator, the emulator and the product library are built (all in-tree)."""
    import __graft_entry__ as g
    g.build()
    return True
