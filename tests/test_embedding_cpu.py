"""CPU checks of the learnable embedding (feature_table.ShardedEmbedding): its lazy row-sparse Adam restated in numpy
is Parameter's update bit for bit, untouched rows keep their bits, the rank-order sum is a left-to-right float32 sum,
and argument errors are raised before any device work."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from embedding_oracle import adam_rows, lazy_adam, rank_order_sum


def _parameter(W, wd=1e-4, lr=0.01, decay=(0.97, 3)):
    from neutronstarlite_b200.toolkits import Parameter
    p = Parameter(W.shape[0], W.shape[1], lr, 0.9, 0.999, 1e-9, wd)
    p.W = torch.from_numpy(W.copy()).requires_grad_(True)
    p.set_decay(*decay)
    return p


def _schedule(wd=1e-4, lr=0.01, decay=(0.97, 3)):
    from neutronstarlite_b200.adam import AdamSchedule
    s = AdamSchedule()
    s._init_schedule(lr, 0.9, 0.999, 1e-9, wd)
    s.set_decay(*decay)
    return s


def test_lazy_adam_touching_every_row_is_the_parameter_host_mirror_bit_for_bit():
    rng = np.random.default_rng(0)
    V, F, steps = 23, 10, 7
    W0 = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    grads = [rng.normal(0, 1e-2, (V, F)).astype(np.float32) for _ in range(steps)]
    p = _parameter(W0, decay=(2, 3))          # a decay rate that survives the reference's int truncation
    for g in grads:
        p.all_reduce_to_gradient(torch.from_numpy(g))
        p.learn_with_decay_Adam()
        p.next()
    W, M, Vm = W0.copy(), np.zeros_like(W0), np.zeros_like(W0)
    lazy_adam(W, M, Vm, [(np.arange(V), g) for g in grads], _schedule(decay=(2, 3)))
    assert np.array_equal(W, p.W.detach().numpy())
    assert np.array_equal(M, p.M.numpy()) and np.array_equal(Vm, p.V.numpy())


def test_lazy_adam_leaves_untouched_rows_alone_and_uses_the_step_wide_schedule():
    """Rows touched at some steps only: untouched rows and moments keep their bits, and a touched row gets exactly
    Parameter's update with the schedule of that step (a one-row Parameter whose schedule advances every step and
    which learns only when its row is touched)."""
    rng = np.random.default_rng(1)
    V, F, steps = 12, 6, 8
    W0 = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    plan = [np.array(sorted(rng.choice(V, size=int(rng.integers(0, 5)), replace=False)), dtype=np.int64)
            for _ in range(steps)]
    plan[2] = np.zeros(0, dtype=np.int64)                     # a step that touches nothing
    grads = [rng.normal(0, 1e-2, (len(ids), F)).astype(np.float32) for ids in plan]
    W, M, Vm = W0.copy(), np.zeros_like(W0), np.zeros_like(W0)
    lazy_adam(W, M, Vm, list(zip(plan, grads)), _schedule())
    for r in range(V):
        p = _parameter(W0[r:r + 1])
        for ids, g in zip(plan, grads):
            hit = np.nonzero(ids == r)[0]
            if hit.size:
                p.all_reduce_to_gradient(torch.from_numpy(g[hit]))
                p.learn_with_decay_Adam()
            p.next()
        assert np.array_equal(W[r], p.W.detach().numpy()[0]), r
        assert np.array_equal(M[r], p.M.numpy()[0]) and np.array_equal(Vm[r], p.V.numpy()[0]), r
    never = np.setdiff1d(np.arange(V), np.concatenate(plan))
    assert never.size > 0
    assert np.array_equal(W[never], W0[never]) and not M[never].any() and not Vm[never].any()


def test_adam_schedule_is_the_one_parameter_steps_with():
    from neutronstarlite_b200.toolkits import Parameter
    from neutronstarlite_b200.adam import AdamSchedule
    assert issubclass(Parameter, AdamSchedule)
    p, s = _parameter(np.zeros((2, 2), np.float32)), _schedule()
    for _ in range(7):
        p.next()
        s.next()
        assert (p.alpha, p.beta1, p.beta2, p.alpha_t) == (s.alpha, s.beta1, s.beta2, s.alpha_t)
    assert s.alpha == 0      # decay rate 0.97 truncates to 0 at the decay epoch, as in the reference


def test_rank_order_sum_is_left_to_right_in_float32():
    a = np.array([1e8, 1.0, -1.0], dtype=np.float32)
    b = np.array([-1e8, 1e-8, 3.0], dtype=np.float32)
    c = np.array([1.0, 2.0, 1e8], dtype=np.float32)
    got = rank_order_sum([a, b, c])
    assert got.dtype == np.float32
    assert np.array_equal(got, ((a + b).astype(np.float32) + c).astype(np.float32))
    assert got[0] == 1.0     # (1e8 - 1e8) + 1, not 1e8 + (-1e8 + 1) = 0 in float32
    assert np.array_equal(rank_order_sum([a]), a)


def test_adam_rows_matches_the_host_mirror_on_one_row():
    rng = np.random.default_rng(2)
    W0 = rng.uniform(-1, 1, (1, 9)).astype(np.float32)
    g = rng.normal(0, 1, (1, 9)).astype(np.float32)
    p = _parameter(W0)
    p.all_reduce_to_gradient(torch.from_numpy(g))
    p.learn_with_decay_Adam()
    W, M, V = W0.copy(), np.zeros_like(W0), np.zeros_like(W0)
    adam_rows(W, M, V, g, _schedule())
    assert np.array_equal(W, p.W.detach().numpy())


# ---- argument errors before any device work ----------------------------------------------------------------------

def _bare(**fields):
    """A ShardedEmbedding without a constructor run: the checks below must raise before they look at anything else."""
    from neutronstarlite_b200.feature_table import ShardedEmbedding
    t = object.__new__(ShardedEmbedding)
    t.__dict__.update(dict(_buf=None, _outbox=None, world=1, rows=10, F=4, capacity=3, device=torch.device("cpu")))
    t.__dict__.update(fields)
    return t


def test_bf16_embedding_is_refused_before_device_work():
    from neutronstarlite_b200._lib import NtsError
    from neutronstarlite_b200.feature_table import ShardedEmbedding
    with pytest.raises(NtsError, match="float32"):
        ShardedEmbedding(torch.zeros(4, 4), [0, 4], dtype=torch.bfloat16)


def test_step_on_a_closed_table_is_refused():
    from neutronstarlite_b200._lib import NtsError
    t = _bare()
    with pytest.raises(NtsError, match="closed"):
        t.step(torch.zeros(1, dtype=torch.int32), torch.zeros(1, 4))
    with pytest.raises(NtsError, match="closed"):
        t._step(torch.zeros(1, dtype=torch.int32), torch.zeros(1, 4))


def test_step_refuses_host_ids_and_more_rows_than_capacity():
    from neutronstarlite_b200._lib import NtsError
    t = _bare(_buf=1)          # "open": no check below may reach the (fake) buffer
    with pytest.raises(NtsError, match="int32"):
        t.step(torch.arange(2, dtype=torch.int32), torch.zeros(2, 4))            # host ids
    with pytest.raises(NtsError, match="capacity"):
        t._step(torch.arange(5, dtype=torch.int32), torch.zeros(5, 4))
