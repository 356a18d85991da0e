"""The levels a strided reverse process visits (`sample(..., steps=K)` of every package).

Algorithm 2 of cold diffusion, x_{t-1} = x_t - D(x0_hat, t) + D(x0_hat, t-1), holds for any pair of levels:
x_s = x_t - D(x0_hat, t) + D(x0_hat, s), s < t.  A K-step sample walks t = tau_0 > tau_1 > ... > tau_K = 0 with
tau_i = round(t (K - i) / K), and each step applies the routine's one-step update with (hi, lo) = (tau_i, tau_{i+1}); the
network still sees hi - 1 as its time input.  K = t visits every level, so it is the full loop."""
import numbers


def reverse_levels(t, steps=None):
    """[tau_0 = t, tau_1, ..., tau_K = 0], strictly decreasing; steps=None -> every level t, t-1, ..., 0.
    Raises ValueError unless steps is None or an integer with 1 <= steps <= t."""
    t = int(t)
    if steps is None:
        return list(range(t, -1, -1))
    if isinstance(steps, bool) or not isinstance(steps, numbers.Integral):
        raise ValueError("steps must be None or an integer, got %r" % (steps,))
    K = int(steps)
    if not 1 <= K <= t:
        raise ValueError("steps must satisfy 1 <= steps <= t = %d, got %d" % (t, K))
    # round half up in integers: floor((2 t (K - i) + K) / 2K)
    return [(2 * t * (K - i) + K) // (2 * K) for i in range(K + 1)]


def refuse_strided(steps, package, routine):
    """the one-step updates of some routines have no strided counterpart: ValueError naming the routine when steps is given"""
    if steps is not None:
        raise ValueError("%s: sample(steps=%r) is not defined for %s; use steps=None" % (package, steps, routine))
