"""CPU restatement of the evaluation pieces (TEST INFRASTRUCTURE -- never imported by ``madrl_b200``):

  * ``eval_episodes``         madrl_eval_episodes_*: the episode records of a rollout cut into launches, bit for bit
                              (every float64 operation rounded on its own, in the kernel's order)
  * ``waterworld_env_action`` heuristics/waterworld.py:11-53 called with one env's Np observations as the batch, as
                              rltools' decrollout calls it (samplers/__init__.py:157): one Frobenius norm for all Np
  * ``reference_statistics``  rltools' evaluate_policy statistics (rltools/rltools/util.py:219-231) from whole episodes'
                              rewards and info sums, with ``discount`` as util.py:56-80 computes it
"""
import numpy as np

CARRY_WORDS, INFO_MAX = 8, 2


def new_carry(E, A):
    return np.zeros((E, A, CARRY_WORDS), np.int64)


def new_records(E, A, C, K):
    """(ret, qsum, len, info_sum) record arrays of K episodes per env, zeroed as the caller allocates them."""
    return (np.zeros((K * E, A)), np.zeros((K * E, A)), np.zeros(K * E, np.int32), np.zeros((K * E, C), np.int64))


def eval_episodes(rew, done, info, discount, K, carry, records):
    """madrl_eval_episodes_* on rew [T, E, A], done [T, E], info [T, E, C] (C = 0 allowed); updates `carry`
    (new_carry) and `records` (new_records) in place.  Elementwise over the (e, a) columns, one step at a time:
    the same float64 operations in the same order as each kernel thread."""
    T, E, A = rew.shape
    C = info.shape[2] if info is not None else 0
    ret_o, qsum_o, len_o, info_o = records
    cd = carry.view(np.float64)
    ret, qsum, G = cd[..., 0].copy(), cd[..., 1].copy(), cd[..., 2].copy()
    ln, k = carry[:, 0, 4].copy(), carry[:, 0, 5].copy()
    pw = np.where(carry[..., 4] == 0, 1.0, cd[..., 3])
    isum = carry[:, 0, 6:6 + INFO_MAX].copy()
    for t in range(T):
        r = rew[t].astype(np.float64)
        ret = ret + r
        G = G + pw
        qsum = qsum + r * G
        pw = pw * discount
        ln += 1
        isum[:, :C] += info[t].astype(np.int64) if C else 0
        end = np.nonzero(done[t])[0]
        keep = end[k[end] < K]
        rec = k[keep] * E + keep
        ret_o[rec], qsum_o[rec], len_o[rec] = ret[keep], qsum[keep], ln[keep]
        info_o[rec] = isum[keep, :C]
        k[end] += 1
        ret[end] = qsum[end] = G[end] = 0.0
        pw[end], ln[end], isum[end] = 1.0, 0, 0
    cd[..., 0], cd[..., 1], cd[..., 2], cd[..., 3] = ret, qsum, G, pw
    carry[..., 4], carry[..., 5] = ln[:, None], k[:, None]
    carry[:, 0, 6:6 + INFO_MAX] = isum
    carry[:, 1:, 6:] = 0


def waterworld_env_action(obs_rows):
    """One env's observations [Np, 7K+2(+1)] -> (actions [Np, 2], the batch's Frobenius norm)
    (heuristics/waterworld.py:25-51 with B = Np; heuristics_oracle.waterworld_action is the B = 1 call)."""
    o = np.asarray(obs_rows, dtype=np.float64)
    K = o.shape[1] // 7                                                     # :26
    ang = np.linspace(0., 2. * np.pi, K + 1)[:-1]                           # :27
    vecs = np.c_[np.cos(ang), np.sin(ang)]                                  # :29
    ob = -np.sum(o[:, 0:K][..., None] * vecs[None], axis=1)                 # :31
    ev = np.sum(o[:, K:2 * K][..., None] * vecs[None], axis=1)              # :34
    po = -np.sum(o[:, 3 * K:4 * K][..., None] * vecs[None], axis=1)         # :37
    pu = np.sum(o[:, 5 * K:6 * K][..., None] * vecs[None], axis=1) / 2      # :40
    ev[o[:, 7 * K] > 0] *= 1.5                                              # :43
    po[o[:, 7 * K + 1] > 0] *= 1.5                                          # :44
    a = ob + ev + po + pu                                                   # :46
    n = np.linalg.norm(a)                                                   # :47
    return (a / n if n > 0 else np.zeros((o.shape[0], 2))), n               # :48-51


def discount(r_N_T, gamma):
    """rltools.util.discount (util.py:56-80) on [N, T]."""
    disc = np.power(gamma, np.arange(r_N_T.shape[1]))
    q = np.cumsum((r_N_T * disc[None])[:, ::-1], axis=1)[:, ::-1]
    return q / disc[None]


def reference_statistics(episodes, disc, mode, info_keys):
    """evaluate_policy's dict from `episodes`: a list of (rewards [L, A], info sums [C]) in record order."""
    A = episodes[0][0].shape[1]
    lmax = max(len(r) for r, _ in episodes)
    infos = {k: np.mean([i[c] for _, i in episodes]) for c, k in enumerate(info_keys)}

    def padded(a):
        return np.array([np.concatenate([r[:, a], np.zeros(lmax - len(r))]) for r, _ in episodes])

    if mode == "centralized":
        r_B_T = padded(0)
        return dict(ret=r_B_T.sum(axis=1).mean(), disc_ret=discount(r_B_T, disc).mean(), **infos)
    rets, stds, discs = [], [], []
    for a in range(A):
        r_B_T = padded(a)
        rets.append(r_B_T.sum(axis=1).mean())
        stds.append(r_B_T.sum(axis=1).std())
        discs.append(discount(r_B_T, disc).mean())
    return dict(ret=np.array(rets), retstd=np.array(stds), disc_ret=np.array(discs),
                **{k: np.full(A, v) for k, v in infos.items()})
