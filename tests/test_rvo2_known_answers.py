"""Analytic known-answer and property tests of the RVO2 restatement (oracle/rvo2_ref.cpp), SURVEY.md §8c.

RVO2 itself is not in the reference checkout (un-vendored, un-pinned `rvo2` = sybrenstuvel/Python-RVO2 bundling the RVO2
Library v2.0.x), so the restatement cannot be diffed against its source here: these cases pin each branch of the
published algorithm on configurations whose answer follows by hand (derivations in the docstrings), and the
end-to-end pin stays the shipped 500-episode logs (tests/test_gpu_eval.py)."""
import math
import os
import sys

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
import rvo2  # noqa: E402

TAU, DT = 5.0, 0.25


def _sim(ego_pos, ego_vel, ego_pref, ego_r=0.5, ego_vmax=1.0, others=(), neighbor_dist=10.0, max_neighbors=None):
    """ego = agent 0 (like orca.py:84-95); others: (pos, vel, radius)."""
    k = len(others) if max_neighbors is None else max_neighbors
    s = rvo2.PyRVOSimulator(DT, neighbor_dist, k, TAU, TAU, ego_r, ego_vmax)
    s.addAgent(tuple(ego_pos), neighbor_dist, k, TAU, TAU, ego_r, ego_vmax, tuple(ego_vel))
    for pos, vel, r in others:
        s.addAgent(tuple(pos), neighbor_dist, k, TAU, TAU, r, 1.0, tuple(vel))
    s.setAgentPrefVelocity(0, tuple(ego_pref))
    for j in range(len(others)):
        s.setAgentPrefVelocity(j + 1, (0.0, 0.0))
    return s


def test_no_neighbours_returns_clamped_preferred_velocity():
    s = _sim((0, 0), (0, 0), (0.5, 0.2))
    s.doStep()
    assert np.allclose(s.getAgentVelocity(0), (0.5, 0.2), atol=1e-7)
    assert s._numLines(0) == 0 and s._lineFail(0) == -1
    s = _sim((0, 0), (0, 0), (3.0, 4.0))              # |pref| = 5 > maxSpeed 1 -> normalised
    s.doStep()
    assert np.allclose(s.getAgentVelocity(0), (0.6, 0.8), atol=1e-6)
    # position integrates the NEW velocity: p += v * dt
    assert np.allclose(s.getAgentPosition(0), (0.15, 0.2), atol=1e-6)


def test_head_on_pair_is_point_symmetric_and_matches_hand_derivation():
    """A (-2,0) -> +x, B (2,0) -> -x, radii 0.5 (R = 1), tau = 5.  For A: relPos = (4,0), relVel = (2,0),
    w = relVel - relPos/tau = (1.2, 0), w.relPos > 0 -> leg case; det(relPos, w) = 0 -> right leg:
    dir = -(4*sqrt15, -4)/16 = (-sqrt15/4, 1/4); u = (relVel.dir) dir - relVel = (-1/8, -sqrt15/8);
    line.point = v + u/2 = (15/16, -sqrt15/16).  pref (1,0) violates the line and its projection on it is the
    line point itself (u is the smallest change), so vA = (15/16, -sqrt15/16); B is the point reflection."""
    others_a = [((2.0, 0.0), (-1.0, 0.0), 0.5)]
    a = _sim((-2.0, 0.0), (1.0, 0.0), (1.0, 0.0), others=others_a)
    a.doStep()
    va = a.getAgentVelocity(0)
    others_b = [((-2.0, 0.0), (1.0, 0.0), 0.5)]
    b = _sim((2.0, 0.0), (-1.0, 0.0), (-1.0, 0.0), others=others_b)
    b.doStep()
    vb = b.getAgentVelocity(0)
    assert np.allclose(va, (15.0 / 16.0, -math.sqrt(15.0) / 16.0), atol=2e-6), va
    # the tie det(relPos, w) == 0 picks the right leg for both agents -> exact point symmetry
    assert va[0] == -vb[0] and va[1] == -vb[1]
    assert a._numLines(0) == 1 and a._lineFail(0) == -1
    px, py, dx, dy = a._line(0, 0)
    assert np.allclose((px, py, dx, dy), (15 / 16, -math.sqrt(15) / 16, -math.sqrt(15) / 4, 0.25), atol=2e-6)


def test_agent_beyond_neighbor_dist_is_ignored():
    far = [((12.0, 0.0), (-1.0, 0.0), 0.5)]           # 12 m away, neighborDist 10
    s = _sim((0, 0), (1.0, 0.0), (1.0, 0.0), others=far, neighbor_dist=10.0)
    s.doStep()
    assert s._numLines(0) == 0
    assert np.allclose(s.getAgentVelocity(0), (1.0, 0.0), atol=1e-7)
    # just inside the range it does produce a line (rangeSq test is strict `<` on the squared distance)
    near = [((9.99, 0.0), (-1.0, 0.0), 0.5)]
    s = _sim((0, 0), (1.0, 0.0), (1.0, 0.0), others=near, neighbor_dist=10.0)
    s.doStep()
    assert s._numLines(0) == 1


def test_overlapping_discs_take_the_collision_branch_with_time_step():
    """Discs overlap (dist 0.5 < R = 1), both at rest: w = relVel - relPos/dt = (-2, 0), unitW = (-1, 0),
    dir = (unitW.y, -unitW.x) = (0, 1), u = (R/dt - |w|) unitW = (4 - 2)(-1, 0) = (-2, 0), line.point = (-1, 0).
    pref (0,0) violates it; its projection on the line x = -1 is (-1, 0), inside maxSpeed 2."""
    s = _sim((0, 0), (0, 0), (0, 0), ego_vmax=2.0, others=[((0.5, 0.0), (0.0, 0.0), 0.5)])
    s.doStep()
    assert np.allclose(s._line(0, 0), (-1.0, 0.0, 0.0, 1.0), atol=1e-6)
    assert np.allclose(s.getAgentVelocity(0), (-1.0, 0.0), atol=1e-6)
    # with the time HORIZON instead of the time step the push would be 20x weaker: the branch matters
    assert abs(s.getAgentVelocity(0)[0]) > 0.9


def test_ring_of_eight_is_infeasible_and_lp3_returns_the_symmetric_optimum():
    """8 neighbours on a ring of radius 1.2 all rushing at the centre at 1.5 m/s: the half-planes exclude every
    velocity (LP2 fails) and linearProgram3 minimises the maximum penetration; by the 8-fold symmetry the
    unique min-max point is the origin."""
    others = []
    for k in range(8):
        ang = 2 * math.pi * k / 8 + 0.1
        c, sn = math.cos(ang), math.sin(ang)
        others.append(((1.2 * c, 1.2 * sn), (-1.5 * c, -1.5 * sn), 0.5))
    s = _sim((0, 0), (0, 0), (0.3, 0.1), others=others)
    s.doStep()
    assert s._numLines(0) == 8
    assert 0 <= s._lineFail(0) < 8                       # LP2 failed at some line -> LP3 ran
    v = s.getAgentVelocity(0)
    assert math.hypot(*v) < 2e-3, v
    # the penetration (signed distance into the forbidden side) is the same for all 8 lines at the optimum
    pen = []
    for k in range(8):
        px, py, dx, dy = s._line(0, k)
        pen.append(dx * (py - v[1]) - dy * (px - v[0]))
    assert max(pen) - min(pen) < 5e-3 and min(pen) > 0


def test_max_neighbors_keeps_the_k_nearest_in_ascending_order():
    dists = [4.0, 1.5, 3.0, 2.0, 6.0, 2.5]
    others = [((d * math.cos(j), d * math.sin(j)), (0.0, 0.0), 0.3) for j, d in enumerate(dists)]
    s = _sim((0, 0), (0, 0), (0.5, 0), ego_r=0.3, others=others, max_neighbors=3)
    s.doStep()
    assert s._neighborIds(0) == [2, 4, 6]                # agent ids 1-based after the ego: d = 1.5, 2.0, 2.5
    assert s._numLines(0) == 3
    # ties: strict `<` in the insertion sort keeps the EARLIER agent first
    others = [((2.0, 0.0), (0, 0), 0.3), ((0.0, 2.0), (0, 0), 0.3), ((-2.0, 0.0), (0, 0), 0.3)]
    s = _sim((0, 0), (0, 0), (0.5, 0), ego_r=0.3, others=others, max_neighbors=3)
    s.doStep()
    assert s._neighborIds(0) == [1, 2, 3]


def _lp3_point_scale(s, n):
    """Largest distance from the origin of the lines linearProgram3 projects for agent 0 (fp64 from its ORCA lines):
    the point of line i moved along it to its intersection with line j, or the midpoint for antiparallel lines."""
    lines = [np.array(s._line(0, k), np.float64) for k in range(n)]
    big = 0.0
    for i in range(max(s._lineFail(0), 0), n):
        pi, di = lines[i][:2], lines[i][2:]
        for j in range(i):
            pj, dj = lines[j][:2], lines[j][2:]
            d = di[0] * dj[1] - di[1] * dj[0]
            if abs(d) <= 1e-5:
                q = 0.5 * (pi + pj)
            else:
                q = pi + ((dj[0] * (pi - pj)[1] - dj[1] * (pi - pj)[0]) / d) * di
            big = max(big, float(np.hypot(*q)))
    return big


def test_lp3_far_projected_line_float32_overshoot():
    """An agent 0.14 m away (overlapping: the collision line) and one 5 m away give two nearly antiparallel ORCA lines
    (det of their directions -0.0037), and line 0 lies 1.39 from the origin, outside the speed circle: LP2 fails there
    and linearProgram3 projects line 1 onto line 0 at |p| = 481.  linearProgram1's discriminant
    dot(p, d)^2 + r^2 - |p|^2 then cancels in float32 and the result lands at |v| = 1.0146 > maxSpeed = 1.  The same
    steps in float64 give (0.95643, -0.29195), on the circle: this is RVO2's own float32 arithmetic, which the oracle
    (and the CUDA environment, bit for bit) reproduce."""
    others = [((5.0, 0.0), (-1.0, 0.0), 0.66), ((0.140625, 0.0), (-0.8125, 1.5), 0.66)]
    s = _sim((0.0, 0.0), (0.0, 0.5), (0.0, 0.0), ego_r=0.535, ego_vmax=1.0, others=others)
    s.doStep()
    assert s._numLines(0) == 2 and s._lineFail(0) == 0
    v = s.getAgentVelocity(0)
    assert v == (np.float32(0.972900390625), np.float32(-0.287872314453125)), v
    assert 1.0145 < math.hypot(*v) < 1.0147
    assert 480 < _lp3_point_scale(s, 2) < 482


# ------------------------------------------------------------------------------------------ property tests
hyp = pytest.importorskip("hypothesis")
from hypothesis import given, settings, strategies as st  # noqa: E402

_coord = st.floats(-5.0, 5.0, allow_nan=False, width=32)
_vel = st.floats(-1.5, 1.5, allow_nan=False, width=32)
_rad = st.floats(0.3125, 0.5, allow_nan=False, width=32)
_other = st.tuples(_coord, _coord, _vel, _vel, _rad)


@settings(max_examples=300, deadline=None)
@given(ego=st.tuples(_coord, _coord, _vel, _vel, _rad, st.floats(0.5, 1.5, width=32), _vel, _vel),
       others=st.lists(_other, min_size=0, max_size=10))
def test_property_speed_limit_and_feasibility(ego, others):
    """(1) |v_new| <= maxSpeed (1 + eps) always; (2) when linearProgram2 succeeds the result satisfies every ORCA
    half-plane: det(dir, point - v) <= eps; (3) with no violated line the result is the clamped preferred velocity."""
    # drop exact coincidences with the ego (RVO2 divides by |w| there)
    others = [o for o in others if (o[0] - ego[0]) ** 2 + (o[1] - ego[1]) ** 2 > 1e-4]
    sim_others = [((o[0], o[1]), (o[2], o[3]), o[4] + 0.16) for o in others]
    s = _sim((ego[0], ego[1]), (ego[2], ego[3]), (ego[6], ego[7]), ego_r=ego[4] + 0.16, ego_vmax=ego[5], others=sim_others)
    s.doStep()
    v = s.getAgentVelocity(0)
    vmax = np.float32(ego[5])
    n = s._numLines(0)
    # (1) holds to rounding when linearProgram2 succeeds; in linearProgram3 RVO2's float32 quadratic on a far projected
    # line may leave the speed circle by up to ~|p| sqrt(eps32) (test_lp3_far_projected_line_float32_overshoot)
    slack = 2.0 * math.sqrt(float(np.finfo(np.float32).eps)) * _lp3_point_scale(s, n) if s._lineFail(0) != -1 else 0.0
    assert math.hypot(*v) <= float(vmax) * (1 + 1e-4) + 1e-6 + slack
    f32 = np.float32
    in_range = sum(1 for o in others
                   if (f32(o[0]) - f32(ego[0])) ** 2 + (f32(o[1]) - f32(ego[1])) ** 2 < f32(100.0))
    assert abs(n - in_range) <= 1                         # (<= 1: a neighbour within one ulp of the 10 m range)
    if s._lineFail(0) == -1:
        for k in range(n):
            px, py, dx, dy = s._line(0, k)
            assert dx * (py - v[1]) - dy * (px - v[0]) <= 2e-4, (k, dx * (py - v[1]) - dy * (px - v[0]))
    # solve_one (the batched helper the oracle env uses) is the same computation
    if others:
        ego_arr = np.array([ego[0], ego[1], ego[2], ego[3], ego[4] + 0.16, ego[5], ego[6], ego[7]], np.float32)
        oth = np.array([[o[0], o[1], o[2], o[3], o[4] + 0.16] for o in others], np.float32)
        vx, vy, nl, fail = rvo2.solve_one(ego_arr, oth, 10.0, TAU, DT)
        assert (vx, vy) == tuple(v) and nl == n and fail == s._lineFail(0)
