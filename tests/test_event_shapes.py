"""CPU: the shape rules of event-shaped sites (distributions._event_layout) and the limits of the event samplers, which
are checked on the host before anything reaches a device."""
import pytest
import torch

from pyprob_b200 import ops
from pyprob_b200.distributions import _event_layout

N = 6


def test_scalar_sites_keep_todays_path():
    assert _event_layout((0.0, 1.0), N, 2.0) is None
    assert _event_layout((torch.zeros(N), 1.0), N, torch.zeros(N)) is None       # [n] value: one per particle
    assert _event_layout((torch.zeros(N, 1), 1.0), N, 0.5) is None               # [n, 1] parameter: one per particle
    assert _event_layout((0.0, 1.0), N, torch.tensor([3.0])) is None             # a 1-element value is a scalar
    assert _event_layout((0.0, 1.0), N) is None


def test_shared_event_of_length_n_is_passed_as_1_by_n():
    E, forms, vform, _ = _event_layout((0.0, 1.0), N, torch.zeros(1, N))
    assert E == (1, N) and vform == 'event'


def test_value_shapes_broadcast_against_parameters():
    E, forms, vform, _ = _event_layout((torch.zeros(28, 1), 1.0), N, torch.zeros(28, 28))
    assert E == (28, 28) and forms[0] == ('event', (28, 1)) and forms[1] == ('scalar', ())
    E, forms, vform, _ = _event_layout((torch.zeros(N, 3), torch.ones(N)), N, torch.zeros(3))
    assert E == (3,) and forms == [('particle_event', (3,)), ('particle', ())]
    E, forms, vform, _ = _event_layout((torch.zeros(1, 4, 5), 1.0), N, 0.0)
    assert E == (4, 5) and vform == 'scalar'
    E, forms, vform, _ = _event_layout((torch.zeros(1, 7), 1.0), N)
    assert E == (7,) and vform is None
    E, forms, vform, _ = _event_layout((0.0, 1.0), N, torch.zeros(N + 1))        # 1-D, not n long: a shared event
    assert E == (N + 1,)
    E, forms, vform, _ = _event_layout((torch.zeros(1, N), 1.0), N, torch.zeros(N))   # [n] under an event parameter
    assert E == (N,) and vform == 'event'


def test_mismatched_shapes_raise_value_error():
    with pytest.raises(ValueError, match='broadcast'):
        _event_layout((torch.zeros(1, 5), 1.0), N, torch.zeros(4))
    with pytest.raises(ValueError, match='broadcast'):
        _event_layout((torch.zeros(1, 5), torch.ones(1, 3)), N)
    with pytest.raises(ValueError, match='broadcast'):
        _event_layout((torch.zeros(N + 1), torch.ones(1, 3)), N)


def test_one_per_particle_parameters_stay_scalar_sites():
    # an [n, 1] parameter (w.view(-1, 1)) with an [n] value: one value per particle, not an n x n event
    assert _event_layout((torch.zeros(N, 1), 1.0), N, torch.zeros(N)) is None
    assert _event_layout((torch.zeros(N, 1, 1), torch.ones(N)), N, torch.zeros(N)) is None
    E, forms, vform, _ = _event_layout((torch.zeros(N, 1), 1.0), N, torch.zeros(3))
    assert E == (3,) and forms[0] == ('particle', ())


def test_one_dimensional_parameter_of_another_length_is_a_shared_event():
    E, forms, vform, _ = _event_layout((torch.zeros(5), 1.0), N, torch.zeros(5))
    assert E == (5,) and forms[0] == ('event', (5,)) and vform == 'event'
    E, forms, vform, _ = _event_layout((torch.zeros(5), 1.0), N, 0.5)
    assert E == (5,) and vform == 'scalar'


def test_sampler_limits_are_host_checks():
    with pytest.raises(ValueError, match='2\\^24'):
        ops.event_sample(0, [0.0, 1.0], 2, (1 << 24) + 1, 1, 1)
    with pytest.raises(ValueError, match='2\\^24'):
        ops.event_sample(0, [0.0, 1.0], 2, 0, 1, 1)
    with pytest.raises(ValueError, match='2\\^40'):
        ops.event_sample(0, [0.0, 1.0], 4, 2, 1, 1, first_index=(1 << 40) - 2)


def test_family_table():
    assert sorted(ops.EVENT_FAMILIES.values()) == list(range(11))
    assert ops.EVENT_NUM_PARAMS[ops.EVENT_FAMILIES['Beta']] == 4
    assert ops.EVENT_NUM_PARAMS[ops.EVENT_FAMILIES['Poisson']] == 1
