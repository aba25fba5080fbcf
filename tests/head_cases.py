"""Case table of the fused Q-head kernel tests (tests/test_head_kernels_gpu.py): shapes, options and data generators of
cb200_dqn_head_fused, cb200_ensemble_head_fused and cb200_c51_head.  Not the cross product: every edge appears at least
once (checked at import by _check_coverage).  numpy only."""
import numpy as np

import head_ref as hr

RULES = [hr.TARGET_DQN, hr.TARGET_MMC, hr.TARGET_PAL, hr.TARGET_PAL_PERSISTENT]
FEATURES = [256, 512]

# ---- DQN head ----------------------------------------------------------------------------------------------------------
DQN_BATCHES = [1, 2, 3, 15, 16, 17, 33, 512, 4096]
DQN_ACTIONS = [1, 2, 3, 6, 7, 8]
# optional outputs: "all" = q_next, loss, q_select / q_target_s and dh; "none" = none of them; "dh" / "planes" / "both"
# = the feature gradient as fp32, as operand planes (batch % 8 == 0 only) or both, the other optional outputs NULL
OUTPUTS = ["all", "none", "dh", "planes", "both"]


def _dqn_cases():
    cases = []
    for i, B in enumerate(DQN_BATCHES):
        for r in RULES:
            k = 4 * i + r
            out = OUTPUTS[k % 5]
            if B % 8 and out in ("planes", "both"):
                out = "dh" if out == "planes" else "all"
            cases.append(dict(rule=r, F=FEATURES[(i + r) % 2], A=DQN_ACTIONS[(i + 2 * r) % 6], B=B,
                              select=r != hr.TARGET_DQN or k % 3 != 0, weights=k % 2 == 0, huber=(k // 2) % 2 == 0,
                              out=out))
    # n_actions 8 at 512 features: 2 * 8 * 512 + 8 * 512 floats = exactly 48 KB of shared memory
    for r, B in zip(RULES, (16, 17, 512, 33)):
        cases.append(dict(rule=r, F=512, A=8, B=B, select=True, weights=r % 2 == 1, huber=r < 2,
                          out="both" if B % 8 == 0 else "all"))
    return cases


DQN_CASES = _dqn_cases()

# ---- ensemble head -------------------------------------------------------------------------------------------------
ENS_HEADS = [1, 2, 10, 64]
ENS_ACTIONS = [1, 6, 8]
ENS_BATCHES = [1, 17, 512]
MASKS = ["random", "zeros", "ones"]


def _ens_cases():
    cases = []
    for i, H in enumerate(ENS_HEADS):
        for j, F in enumerate(FEATURES):
            k = 2 * i + j
            B = ENS_BATCHES[k % 3]
            cases.append(dict(H=H, F=F, A=ENS_ACTIONS[(k + i) % 3], B=B, masks=MASKS[k % 3],
                              rescale=(1.0, 0.1)[(k // 3) % 2], huber=k % 2 == 0,
                              out=("both" if B % 8 == 0 else "dh") if k % 4 != 3 else "none"))
    cases.append(dict(H=64, F=512, A=8, B=512, masks="random", rescale=0.1, huber=True, out="planes"))
    cases.append(dict(H=10, F=512, A=6, B=17, masks="ones", rescale=1.0, huber=False, out="all"))
    return cases


ENS_CASES = _ens_cases()

# ---- C51 ---------------------------------------------------------------------------------------------------------------
C51_ATOMS = [2, 3, 31, 32, 33, 51, 64, 101, 768, 769, 1024]
C51_ACTIONS = [1, 2, 6, 18]
C51_BATCHES = [1, 3, 4, 5, 33, 512]
SUPPORTS = [(-10.0, 10.0), (-5.0, 5.0), (0.0, 1.0), (-1.0, 3.0), (-100.0, 100.0)]
LOGITS = ["normal", "extreme", "equal"]


def _c51_cases():
    cases = []
    for i, N in enumerate(C51_ATOMS):
        for j in range(2):
            k = 2 * i + j
            A = C51_ACTIONS[k % 4]
            B = C51_BATCHES[k % 6]
            if N >= 768 and A * B > 600:                # keep the large-support cases' host reference quick
                B = 5
            cases.append(dict(N=N, A=A, B=B, support=SUPPORTS[k % 5], next_is_prob=k % 2,
                              select=(k // 2) % 2 == 1, bootstrap=(k // 3) % 2 == 1, logits=LOGITS[k % 3]))
    # the preset's shape, and the supports whose top bin position rounds above N - 1 with large batches
    cases.append(dict(N=51, A=6, B=512, support=(-10.0, 10.0), next_is_prob=0, select=False, bootstrap=False,
                      logits="normal"))
    cases.append(dict(N=101, A=2, B=512, support=(-10.0, 10.0), next_is_prob=1, select=False, bootstrap=False,
                      logits="normal"))
    cases.append(dict(N=1024, A=2, B=33, support=(-10.0, 10.0), next_is_prob=1, select=True, bootstrap=True,
                      logits="normal"))
    for c in cases:
        c["guard"] = bool(hr.projection_overflow(np.linspace(c["support"][0], c["support"][1], c["N"])))
    return cases


C51_CASES = _c51_cases()


def case_id(c):
    return "-".join("%s%s" % (k, v if not isinstance(v, tuple) else "%g_%g" % v) for k, v in sorted(c.items()))


def _check_coverage():
    seen = lambda key, cases: {c[key] for c in cases}                                          # noqa: E731
    assert seen("B", DQN_CASES) >= set(DQN_BATCHES) and seen("A", DQN_CASES) >= set(DQN_ACTIONS)
    assert {(c["rule"], c["F"]) for c in DQN_CASES} == {(r, f) for r in RULES for f in FEATURES}
    assert {(c["F"], c["A"]) for c in DQN_CASES} >= {(f, a) for f in FEATURES for a in DQN_ACTIONS}
    for key, vals in (("select", (False, True)), ("weights", (False, True)), ("huber", (False, True)),
                      ("out", OUTPUTS)):
        assert seen(key, DQN_CASES) >= set(vals), key
    assert seen("H", ENS_CASES) >= set(ENS_HEADS) and seen("A", ENS_CASES) >= set(ENS_ACTIONS)
    assert seen("B", ENS_CASES) >= set(ENS_BATCHES) and seen("masks", ENS_CASES) >= set(MASKS)
    assert seen("rescale", ENS_CASES) >= {1.0, 0.1} and seen("F", ENS_CASES) >= set(FEATURES)
    assert seen("N", C51_CASES) >= set(C51_ATOMS) and seen("A", C51_CASES) >= set(C51_ACTIONS)
    assert seen("B", C51_CASES) >= set(C51_BATCHES) and seen("logits", C51_CASES) >= set(LOGITS)
    for key in ("next_is_prob", "select", "bootstrap", "guard"):
        assert seen(key, C51_CASES) >= {False, True}, key


_check_coverage()


# ---- data ----------------------------------------------------------------------------------------------------------
def _actions(rng, B, A, out_of_range):
    a = rng.randint(0, A, B).astype(np.int64)
    if out_of_range and B > 2:
        a[1], a[B // 2] = A, -1                             # outside [0, A): the row keeps Q(s), td_err = 0
    return a


def dqn_planted(c, seed=0):
    """Q values planted through h = [Q | 0], W = [I; 0], b = 0: multiples of 1/64 with argmax ties, terminal rows whose
    reward puts e at exactly 0 and +-1 (the Huber kink), and out-of-range actions"""
    rng = np.random.RandomState(seed)
    B, A, F = c["B"], c["A"], c["F"]
    q = {k: (rng.randint(-256, 257, (B, A)) / 64.0).astype(np.float32) for k in ("online", "next", "select", "target_s")}
    for k in ("select", "next", "target_s"):
        q[k][::3] = q[k][::3].max(axis=1, keepdims=True)      # every third row: all actions tie (first maximum wins)
    if A > 2:
        q["select"][1::3, A - 1] = q["select"][1::3, 0] = q["select"][1::3].max(axis=1) + 1   # a two-way tie
    act = _actions(rng, B, A, True)
    done = (rng.rand(B) < 0.5).astype(np.uint8)
    ai = np.clip(act, 0, A - 1)
    qa = q["online"][np.arange(B), ai].astype(np.float64)
    kind = np.arange(B) % 4
    rewards = rng.randint(-64, 65, B) / 16.0
    done[kind < 3] = 1
    rewards = np.where(kind == 0, qa, np.where(kind == 1, qa - 1.0, np.where(kind == 2, qa + 1.0, rewards)))

    def feat(x):
        h = np.zeros((B, F), np.float32)
        h[:, :A] = x
        return h
    eye = np.zeros((F, A), np.float32)
    eye[:A] = np.eye(A, dtype=np.float32)
    zero = np.zeros(A, np.float32)
    return dict(h_next=feat(q["next"]), h_online=feat(q["online"]), h_select=feat(q["select"]),
                h_target_s=feat(q["target_s"]), w_target=eye, b_target=zero, w_online=eye, b_online=zero.copy(),
                actions=act, rewards=rewards, game_overs=done, returns=rng.randint(-64, 65, B) / 16.0,
                weights=rng.choice([0.5, 1.0, 2.0], B).astype(np.float32), discount=0.99, alpha=0.75, rho=0.25)


def dqn_dyadic(c, seed=1):
    """small dyadic h, W, b, rewards, returns and weights (h in {0, 1/2, 1} with three nonzeros a row, W and b in
    {-1/2, 0, 1/2}, discount, alpha and rho 1/2) so that every product and partial sum of the head is exact in fp32
    when the batch is a power of two (then 1 / B is too)"""
    rng = np.random.RandomState(seed)
    B, A, F = c["B"], c["A"], c["F"]

    def feat():
        h = np.zeros((B, F), np.float32)
        for b in range(B):
            h[b, rng.choice(F, 3, replace=False)] = rng.choice([0.5, 1.0], 3)
        return h
    w = lambda: (rng.randint(-1, 2, (F, A)) / 2.0).astype(np.float32)                          # noqa: E731
    return dict(h_next=feat(), h_online=feat(), h_select=feat(), h_target_s=feat(), w_target=w(),
                b_target=(rng.randint(-1, 2, A) / 2.0).astype(np.float32), w_online=w(),
                b_online=(rng.randint(-1, 2, A) / 2.0).astype(np.float32), actions=_actions(rng, B, A, False),
                rewards=rng.randint(-8, 9, B) / 8.0, game_overs=(rng.rand(B) < 0.3).astype(np.uint8),
                returns=rng.randint(-8, 9, B) / 8.0, weights=rng.choice([0.5, 1.0], B).astype(np.float32),
                discount=0.5, alpha=0.5, rho=0.5)


def dqn_random(c, seed=2):
    rng = np.random.RandomState(seed)
    B, A, F = c["B"], c["A"], c["F"]
    feat = lambda: np.maximum(rng.randn(B, F), 0).astype(np.float32)                          # noqa: E731
    return dict(h_next=feat(), h_online=feat(), h_select=feat(), h_target_s=feat(),
                w_target=(rng.randn(F, A) * 0.05).astype(np.float32), b_target=(rng.randn(A) * 0.1).astype(np.float32),
                w_online=(rng.randn(F, A) * 0.05).astype(np.float32), b_online=(rng.randn(A) * 0.1).astype(np.float32),
                actions=_actions(rng, B, A, True), rewards=rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], B),
                game_overs=(rng.rand(B) < 0.2).astype(np.uint8), returns=rng.randn(B) * 3,
                weights=rng.uniform(0.1, 1.0, B).astype(np.float32), discount=0.99, alpha=0.7, rho=0.3)


def ens_data(c, seed=3, dyadic=False):
    rng = np.random.RandomState(seed)
    B, A, F, H = c["B"], c["A"], c["F"], c["H"]
    if dyadic:
        feat = lambda: (rng.randint(0, 3, (B, F)) * (rng.rand(B, F) < 4.0 / F) / 2.0).astype(np.float32)  # noqa: E731
        w = lambda: (rng.randint(-1, 2, (F, H * A)) / 2.0).astype(np.float32)                 # noqa: E731
        b = lambda: (rng.randint(-1, 2, H * A) / 2.0).astype(np.float32)                      # noqa: E731
        rewards, discount = rng.randint(-8, 9, B) / 8.0, 0.5
    else:
        feat = lambda: np.maximum(rng.randn(B, F), 0).astype(np.float32)                      # noqa: E731
        w = lambda: (rng.randn(F, H * A) * 0.05).astype(np.float32)                           # noqa: E731
        b = lambda: (rng.randn(H * A) * 0.1).astype(np.float32)                               # noqa: E731
        rewards, discount = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], B), 0.99
    masks = {"random": (rng.rand(B, H) < 0.5), "zeros": np.zeros((B, H), bool), "ones": np.ones((B, H), bool)}
    return dict(h_next=feat(), h_online=feat(), h_select=feat(), w_target=w(), b_target=b(), w_online=w(),
                b_online=b(), actions=rng.randint(0, A, B).astype(np.int64), rewards=rewards,
                game_overs=(rng.rand(B) < 0.2).astype(np.uint8), masks=masks[c["masks"]].astype(np.uint8),
                discount=discount)


def c51_data(c, seed=4):
    """logits: "normal" (scale 2), "extreme" (+-80: the softmax underflows to exact zeros) or "equal" (every other row
    all equal, a uniform distribution; equal rows across actions also tie the target action).  Rewards hit the clamp
    at both ends and land terminal samples on grid points (an integral b_j credits nothing)."""
    rng = np.random.RandomState(seed)
    B, A, N = c["B"], c["A"], c["N"]
    z = np.linspace(c["support"][0], c["support"][1], N)

    def logits():
        if c["logits"] == "extreme":
            x = rng.choice([-80.0, 80.0, 0.0], (B, A, N), p=[0.45, 0.1, 0.45])
        else:
            x = rng.randn(B, A, N) * 2
            if c["logits"] == "equal":
                x[::2] = 0.5
        return x.astype(np.float32)
    nxt, online, select = logits(), logits(), logits()
    if A > 1:
        nxt[1::4, 1] = nxt[1::4, 0]                           # two actions with the same distribution: a tie
        select[1::4, 1] = select[1::4, 0]
    if c["next_is_prob"]:
        nxt, select = hr.softmax32(nxt), hr.softmax32(select)
    kind = np.arange(B) % 4
    span = z[-1] - z[0]
    rewards = np.where(kind == 0, z[-1] + span, np.where(kind == 1, z[0] - span,
                       np.where(kind == 2, z[rng.randint(0, N, B)], rng.uniform(z[0], z[-1], B))))
    done = (kind == 2) | (rng.rand(B) < 0.2)
    bootstrap = np.where(done, 0.0, rng.choice([1.0, 0.5], B))
    return dict(next=nxt, online=online, select=select if c["select"] else None,
                actions=rng.randint(0, A, B).astype(np.int64), rewards=rewards,
                game_overs=done.astype(np.uint8), bootstrap=bootstrap if c["bootstrap"] else None, z=z,
                gamma_n=0.99)
