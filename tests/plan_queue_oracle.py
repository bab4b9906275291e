"""Faster's committed plan (plan_, faster.hpp:70) restated with collections.deque: updateState's first push, choosing A,
getNextGoal and appendToPlan with its early return, as fq_queue_* and fq_replan_pairs_queue* keep it on rings.  Every state
is a 12-double row (pos vel accel jerk).  Only tests/ and tools/ import it."""
import collections

import numpy as np

QUEUE_OK, QUEUE_NONE, QUEUE_PUBLISHED, QUEUE_CAPACITY, QUEUE_ROWS = 0, 1, 2, 3, 4   # FQ_QUEUE_*
DELTA_T = 10                                                                         # deltaT_, faster.hpp:131


def reset(pos):
    """updateState while uninitialised (faster.cpp:253-266): one state holding only pos."""
    s = np.zeros(12)
    s[:3] = pos
    return collections.deque([s])


def select(plan, delta_t=DELTA_T):
    """faster.cpp:350-352.  -> (x0 (9: A's pos vel accel), k_end_whole); an empty plan gives (NaN, -1)."""
    if not plan:
        return np.full(9, np.nan), -1
    k = max(len(plan) - delta_t, 0)
    return plan[len(plan) - 1 - k][:9].copy(), k


def pop(plan, ticks):
    """getNextGoal (faster.cpp:699-723) `ticks` times: the front, popped while more than one state is left.  -> goals."""
    goals = []
    for _ in range(ticks):
        goals.append(plan[0].copy() if plan else np.full(12, np.nan))
        if len(plan) > 1:
            plan.popleft()
    return np.array(goals).reshape(ticks, 12)


def append(plan, k_end, piece, cap):
    """appendToPlan (faster.cpp:606-648) of `piece` (rows x 12, or None: the replan returned before it) with size read
    now; cap: the ring's capacity.  -> status; the plan changes only on QUEUE_OK."""
    if piece is None or len(piece) == 0 or k_end < 0:
        return QUEUE_NONE
    if len(plan) - 1 - k_end < 0:
        return QUEUE_PUBLISHED                                   # "Already publised the point A"
    keep = len(plan) - 1 - k_end
    if keep + len(piece) > cap:
        return QUEUE_CAPACITY
    for _ in range(k_end + 1):
        plan.pop()
    plan.extend(np.array(row, np.float64) for row in piece)
    return QUEUE_OK


def goal_seen(plan, G, goal_radius):
    """faster.cpp:563-572: |G_term - plan_.back().pos| < goal_radius, the norm as sqrt((dx^2 + dy^2) + dz^2)."""
    d = np.asarray(G, np.float64) - plan[-1][:3]
    return bool(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) < goal_radius)


def to_ring(plans, cap, heads=None):
    """Ring arrays (states n_rows x cap x 12, head, size) holding `plans`, row r's front at heads[r] (default 0); unused
    slots are 0."""
    n = len(plans)
    heads = np.zeros(n, np.int32) if heads is None else np.asarray(heads, np.int32)
    ring = dict(states=np.zeros((n, cap, 12)), head=heads.copy(), size=np.array([len(p) for p in plans], np.int32))
    for r, p in enumerate(plans):
        for i, s in enumerate(p):
            ring["states"][r, (heads[r] + i) % cap] = s
    return ring


def from_ring(ring, r):
    """Row r of a ring as a deque."""
    cap = ring["states"].shape[1]
    return collections.deque(ring["states"][r][(int(ring["head"][r]) + i) % cap].copy() for i in range(int(ring["size"][r])))
