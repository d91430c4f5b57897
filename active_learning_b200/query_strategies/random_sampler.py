from .strategy import Strategy


class RandomSampler(Strategy):
    """active_learning/src/query_strategies/random_sampler.py: the first `budget` entries of the
    shuffled pool.  Host-only (no scoring arithmetic); kept because it is `--strategy`'s default."""

    def query(self, budget):
        pool = self.available_query_idxs()
        picked = [idx for _, idx in zip(range(int(budget)), pool)]
        return picked, max(len(picked), 1)
