"""Host side of disvae.data.DeviceLoader: the epoch plan (padding, each rank's batch windows, the number of batches)
and the check that only ToTensor images of bytes are stored as uint8."""
import pytest
import torch

from disvae.data import batch_windows, padded_length, quantize_unit_bytes


@pytest.mark.parametrize("n", [1, 5, 63, 64, 65, 1000, 1023])
@pytest.mark.parametrize("b", [1, 7, 64])
@pytest.mark.parametrize("drop_last", [False, True])
def test_single_process_plan_is_the_dataloaders(n, b, drop_last):
    batches = list(torch.utils.data.DataLoader(list(range(n)), batch_size=b, drop_last=drop_last))
    w = batch_windows(n, b, drop_last=drop_last)
    assert len(w) == len(batches)
    assert [list(range(s, s + k)) for s, k in w] == [x.tolist() for x in batches]
    assert padded_length(n, 1, drop_last) == n


@pytest.mark.parametrize("n,b,world", [(1003, 16, 2), (1003, 16, 4), (1000, 10, 4), (7, 2, 2), (5, 4, 3), (1, 8, 2),
                                       (64, 8, 8)])
@pytest.mark.parametrize("drop_last", [False, True])
def test_data_parallel_plan(n, b, world, drop_last):
    total = padded_length(n, world, drop_last)
    assert total % world == 0
    assert total == (-(-n // world) * world if not drop_last else n // world * world)
    plans = [batch_windows(n, b, world, r, drop_last) for r in range(world)]
    assert all(len(p) == len(plans[0]) for p in plans)
    pos = 0
    for step in range(len(plans[0])):
        sizes = {p[step][1] for p in plans}
        assert len(sizes) == 1                                            # equal shards at every step
        size = sizes.pop()
        assert 1 <= size <= b
        for r in range(world):                                            # rank-major blocks of one global batch
            assert plans[r][step][0] == pos + r * size
        pos += world * size
    if drop_last:
        assert pos == total // (world * b) * world * b
        assert len(plans[0]) == n // (world * b)
    else:
        assert pos == total                                               # the padded order, covered once
        assert len(plans[0]) == -(-total // (world * b))


def test_k255_check_accepts_totensor_bytes_and_names_the_item():
    k = torch.arange(256, dtype=torch.uint8).view(4, 1, 8, 8)
    x = k.float().div(255)
    assert torch.equal(quantize_unit_bytes(x), k)
    for bad_value in (0.5, 1.0 + 1 / 255, -1 / 255, float("nan"), 2.0, 0.1):
        y = x.clone()
        y[2, 0, 3, 3] = bad_value
        with pytest.raises(RuntimeError, match="item 12 "):
            quantize_unit_bytes(y, first_index=10)
    y = x.clone()
    y[1, 0, 0, 0] = torch.nextafter(y[1, 0, 0, 0], torch.tensor(1.0))   # one ulp off k/255
    with pytest.raises(RuntimeError, match="item 1 "):
        quantize_unit_bytes(y)
    with pytest.raises(RuntimeError, match="float64"):
        quantize_unit_bytes(x.double())
    normalised = (x - 0.5) / 0.5
    with pytest.raises(RuntimeError, match="item 0 "):
        quantize_unit_bytes(normalised)
