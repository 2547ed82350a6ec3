"""The slot exchange of the row-owner pivot search (csrc/panel.cu, grids of <= 32 CTAs) as a CPU model
(oracle/panel_exchange_ref.py): randomised interleavings of publish / gather / barrier with the two-parity slots and the
epoch rule.  No slot word may be overwritten before every reader of its column has read it, every gather completes, and
every CTA sees the same winner and row."""
import pytest

from oracle import panel_exchange_ref as px


@pytest.mark.parametrize("G", [1, 2, 3, 8, 32])
def test_exchange_is_safe_in_every_sampled_interleaving(G):
    ncols = 7 if G < 32 else 4
    for seed in range(40 if G < 32 else 6):
        out = px.run(G, ncols, seed)
        assert out[0] == px.expected(G, ncols)


def test_epoch_carries_over_between_launches_on_one_workspace():
    for seed in range(20):
        out = px.run(5, 6, seed, launches=3)
        for launch in range(3):
            assert out[launch] == px.expected(5, 6, launch=launch)
    # odd column counts keep the base even, so slot parity stays column parity
    out = px.run(4, 5, 1, launches=2)
    assert out[1] == px.expected(4, 5, launch=1)


def test_publishing_ahead_of_the_gather_is_caught():
    """Publishing the next column before this CTA's gather has completed reuses a slot other CTAs may still read."""
    caught = 0
    for seed in range(40):
        try:
            px.run(4, 7, seed, early_publish=True)
        except px.ExchangeError:
            caught += 1
    assert caught > 0
    with pytest.raises(px.ExchangeError):
        for seed in range(40):
            px.run(4, 7, seed, early_publish=True)
