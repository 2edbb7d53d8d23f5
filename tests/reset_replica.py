"""numpy replica of the batched episode reset (csrc/reset_core.h, csrc/reset.cu): Philox4x32-10 over numpy integers and the sequential
rejection sampler, candidate by candidate, in fp32 with every operation rounded on its own.  The GPU tests compare the kernel with it
bit for bit; the CPU tests check its constraints and its Philox against CUDA's."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
OBSTACLES, AGENTS, GOALS, HEADINGS = 0, 1, 2, 3
TWO_PI = np.float32(6.28318548202514648)
PI = np.float32(3.14159274101257324)
ENVS = {'SimpleCar': (2, 4), 'DubinsCar': (2, 4), 'SimpleDrone': (3, 6)}       # pos_dim, state_dim


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of counters (c0..c3) under key (k0, k1); numpy integer arrays broadcast, returns four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0 & MASK), np.uint64(k1 & MASK)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(W0)) & np.uint64(MASK), (k1 + np.uint64(W1)) & np.uint64(MASK)
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & np.uint64(MASK), (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & np.uint64(MASK)]
    return [x.astype(np.uint32) for x in c]


def uniforms(seed, env, episode, tag, ks):
    """[len(ks), 4] fp32 uniforms of draws ks of stream `tag`: (word >> 8) * 2^-24."""
    ks = np.asarray(ks, dtype=np.uint64)
    w = philox(ks, env, episode, tag, seed & MASK, (seed >> 32) & MASK)
    return np.stack([(x >> 8).astype(np.float32) * np.float32(2.0 ** -24) for x in w], axis=1)


def dist2(p, c):
    """sum_d (p_d - c_d)^2 for rows p [k, dim] against one point c, d ascending, fp32, each operation rounded."""
    s = np.zeros(p.shape[0], dtype=np.float32)
    for d in range(p.shape[1]):
        diff = p[:, d] - c[d]
        s = s + diff * diff
    return s


def place(seed, env, episode, tag, count, dim, side, min_dist2, obs=None, clear2=0.0, max_tries=200000, chunk=256):
    """The sequential sampler: candidates k = 0, 1, ... of the stream; c is accepted unless dist2 <= min_dist2 to a placed point or
    <= clear2 to an obstacle.  Returns (points [count, dim] fp32, ok)."""
    side, md2, cl2 = np.float32(side), np.float32(min_dist2), np.float32(clear2)
    pts = np.zeros((count, dim), dtype=np.float32)
    i, k = 0, 0
    while i < count:
        if k >= max_tries:
            return pts, False
        ks = np.arange(k, min(k + chunk, max_tries))
        cands = uniforms(seed, env, episode, tag, ks)[:, :dim] * side
        for c in cands:
            k += 1
            if i and (dist2(pts[:i], c) <= md2).any():
                continue
            if obs is not None and len(obs) and (dist2(obs, c) <= cl2).any():
                continue
            pts[i] = c
            i += 1
            if i == count:
                break
    return pts, True


def reset_env(env_name, spec, n, seed, env, episode, max_tries=200000):
    """One env's reset as gcbf_env_reset_batch draws it: (states [n + num_obs, state_dim], goals [n, goal_dim], failed code)."""
    pd, sd = ENVS[env_name]
    o, gd = spec['num_obs'], spec['goal_dim']
    states = np.zeros((n + o, sd), dtype=np.float32)
    goals = np.zeros((n, gd), dtype=np.float32)
    area = np.float32(spec['area'])
    if o:
        u = uniforms(seed, env, episode, OBSTACLES, np.arange(o))
        states[n:, :pd] = u[:, :pd] * area
        if env_name == 'DubinsCar':
            states[n:, 2] = u[:, 2] * TWO_PI
            states[n:, 3] = u[:, 3] * np.float32(spec['obs_speed_limit'])
    obs = states[n:, :pd]
    agents, ok = place(seed, env, episode, AGENTS, n, pd, area, spec['agent_dist2'], obs, spec['clear2'], max_tries)
    if not ok:
        return states, goals, 1
    states[:n, :pd] = agents
    heads = uniforms(seed, env, episode, HEADINGS, np.arange(n))
    if env_name == 'DubinsCar':
        states[:n, 2] = heads[:, 0] * TWO_PI - PI
    gl, ok = place(seed, env, episode, GOALS, n, pd, area, spec['goal_dist2'], obs, spec['clear2'], max_tries)
    if not ok:
        return states, goals, 2
    goals[:, :pd] = gl
    if env_name == 'DubinsCar' and gd > 2:
        goals[:, 2] = heads[:, 1] * TWO_PI - PI
    return states, goals, 0


def check_constraints(env_name, spec, n, states, goals, atol=0.0):
    """Assertion messages (empty list: all hold) for one env's reset: box, spacing, clearance, heading range, zero velocities."""
    pd, sd = ENVS[env_name]
    o = spec['num_obs']
    bad = []
    area = np.float32(spec['area'])
    for name, pts, md2 in (('agents', states[:n, :pd], spec['agent_dist2']), ('goals', goals[:, :pd], spec['goal_dist2'])):
        if (pts < 0).any() or (pts >= area).any():
            bad.append(f'{name} outside the box')
        for i in range(1, n):
            if (dist2(pts[:i], pts[i]) <= np.float32(md2)).any():
                bad.append(f'{name} spacing')
                break
        for j in range(o):
            if (dist2(pts, states[n + j, :pd]) <= np.float32(spec['clear2'])).any():
                bad.append(f'{name} obstacle clearance')
                break
    if o and ((states[n:, :pd] < 0).any() or (states[n:, :pd] >= area).any()):
        bad.append('obstacles outside the box')
    if env_name == 'DubinsCar':
        for name, h in (('agent heading', states[:n, 2]), ('goal heading', goals[:, 2])):
            if (h < -PI).any() or (h >= PI).any():
                bad.append(f'{name} range')
        if (states[:n, 3] != 0).any():
            bad.append('agent speed')
        if o and ((states[n:, 2] < 0).any() or (states[n:, 2] >= TWO_PI).any() or (states[n:, 3] < 0).any()
                  or (states[n:, 3] >= np.float32(spec['obs_speed_limit'])).any()):
            bad.append('obstacle heading / speed range')
    else:
        if (states[:, pd:] != 0).any():
            bad.append('velocities')
        if (goals[:, pd:] != 0).any():
            bad.append('goal padding')
    return bad
