"""GPU: graphs.GraphCache.upload, the per-step host rows a captured graph reads from its home buffer."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_upload_feeds_a_captured_graph_the_latest_rows(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from baselines_b200 import _lib, graphs
    monkeypatch.setenv("B200RL_NO_GRAPHS", "0")
    cache = graphs.GraphCache()
    dev = torch.device("cuda", torch.cuda.current_device())
    out = torch.zeros(8, 3, dtype=torch.int64, device=dev)
    rng = np.random.RandomState(0)
    r0 = _lib.REPLAYS
    # three uploads alternate the two pinned buffers; the first call runs eagerly, the second captures and replays,
    # the third replays the graph captured over the home, which must read the third upload's rows
    for _ in range(3):
        rows = rng.randint(-2 ** 40, 2 ** 40, (5, 3)).astype(np.int64)
        sel = cache.upload("sel", rows, 8, (3,), torch.int64, dev)
        cache.run(("copy",), lambda: out[:5].copy_(sel))
        assert np.array_equal(out[:5].cpu().numpy(), rows)
    assert _lib.REPLAYS - r0 == 2
    with pytest.raises(ValueError):
        cache.upload("sel", np.zeros((9, 3), np.int64), 8, (3,), torch.int64, dev)
