"""The crafted trie corpus (tests/trie_edges.py) on the CPU: the two CPU statements of mptize agree on every case, every case
reaches the edges it names, and the corpus as a whole keeps each edge above its floor."""
import trie_edges
from helpers import py_mptize


def test_two_cpu_statements_agree_on_every_case(oracle):
    for case in trie_edges.corpus():
        assert py_mptize(oracle.keccak256, case.kv) == oracle.mptize(case.kv), case.name


def test_every_case_reaches_its_targets(oracle):
    for case in trie_edges.corpus():
        got = trie_edges.labels(trie_edges.classify(oracle.keccak256, case.kv))
        missing = [t for t in case.targets if not got[t]]
        assert not missing, (case.name, missing)


def test_edge_floors(oracle):
    counts = trie_edges.reached(oracle.keccak256, trie_edges.corpus())
    for target, floor in sorted(trie_edges.TARGET_FLOORS.items(), key=str):
        print(f"{' / '.join(map(str, target)):40s} {counts[target]:4d}  (floor {floor})")
    low = {t: (counts[t], f) for t, f in trie_edges.TARGET_FLOORS.items() if counts[t] < f}
    assert not low, low
