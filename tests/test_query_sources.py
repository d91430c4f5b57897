"""The host protocol of the samplers that pick from CoreSet's pool, read from their sources.

Each of these samplers is held bit for bit to an oracle and to NumPy's RNG state, so the pool (its two shuffles), the
budget clamp and the random fill must not exist in more than one spelling: they are written once, in coreset.py's
PoolQuery, and a new sampler inherits them instead of copying them."""
import os

QS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "active_learning_b200", "query_strategies")


def _sources():
    out = {}
    for name in sorted(os.listdir(QS)):
        if name.endswith(".py"):
            with open(os.path.join(QS, name)) as f:
                out[name] = f.read()
    return out


def test_only_coreset_builds_the_pool():
    assert [n for n, s in _sources().items() if "get_idxs_for_coreset(" in s] == ["coreset.py"]


def test_the_random_fill_is_written_once():
    assert sum(s.count("np.random.choice(np.flatnonzero(") for s in _sources().values()) == 1
