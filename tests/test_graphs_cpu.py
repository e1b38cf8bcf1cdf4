"""graphs.GraphCache.home: the fixed buffers captured graphs read.  A request that fits returns the same buffer and
keeps the graphs; one that needs a new buffer drops every graph and the seen set, so no graph replays over the
buffer it replaced."""
import torch

from baselines_b200 import graphs


def _cache_with_entries():
    cache = graphs.GraphCache()
    buf = cache.home("obs", 8, (4, 3), torch.uint8, "cpu")
    cache.graphs[("act", 8)] = (object(), 7)
    cache.seen.update({("act", 8), ("act", 4)})
    return cache, buf


def test_first_home_keeps_the_graphs():
    cache = graphs.GraphCache()
    cache.graphs[("train", 4)] = (object(), 3)
    cache.seen.add(("train", 4))
    buf = cache.home("idx", 16, (), torch.int64, "cpu")
    assert buf.shape == (16,) and buf.dtype == torch.int64 and not buf.any()
    assert ("train", 4) in cache.graphs and ("train", 4) in cache.seen


def test_a_request_that_fits_keeps_the_buffer_and_the_graphs():
    cache, buf = _cache_with_entries()
    for rows in (8, 5, 1):
        assert cache.home("obs", rows, torch.Size([4, 3]), torch.uint8, "cpu") is buf
    assert ("act", 8) in cache.graphs and cache.seen == {("act", 8), ("act", 4)}
    # another name is another buffer; allocating it replaces nothing
    assert cache.home("idx", 8, (), torch.int64, "cpu") is not buf
    assert ("act", 8) in cache.graphs and len(cache.seen) == 2


def test_growth_or_another_shape_or_dtype_reallocates_and_drops_the_graphs():
    for rows, trailing, dtype in ((9, (4, 3), torch.uint8), (8, (4, 4), torch.uint8), (8, (12,), torch.uint8),
                                  (8, (4, 3), torch.float32)):
        cache, buf = _cache_with_entries()
        new = cache.home("obs", rows, trailing, dtype, "cpu")
        assert new is not buf and new.shape == (rows,) + trailing and new.dtype == dtype
        assert cache.graphs == {} and cache.seen == set()
        assert cache.home("obs", rows, trailing, dtype, "cpu") is new         # the new buffer is the home from now on
