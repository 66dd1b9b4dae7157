"""Writes tests/golden/fs_odom_golden.json: an independent plain-Python restatement (glibc libm through the math module) of FastSLAM's
odometry motion model (include/fs_odom_math.h, DESIGN §3.15): the increment, FastSLAM 1.0's move, the proposal's prior and FastSLAM
2.0's pose in each of its three cases, on fixed inputs with injected normals.  tests/test_fs_odom_oracle.py checks that the glibc
build of tests/host/fs_odom_oracle.c reproduces every value bit for bit.  Run: python tests/golden/make_fs_odom_golden.py"""
import json
import math
import os

PI = 3.141592653589793
EPS = 1e-8
R00, R11 = 0.5, 0.0305


def wrap(a):
    while a > PI:
        a -= 2.0 * PI
    while a < -PI:
        a += 2.0 * PI
    return a


def rot_noise(a):
    d1, d2 = abs(wrap(a)), abs(wrap(a - PI))
    return d2 if d2 < d1 else d1


def increment(o, al):
    dx, dy = o[3] - o[0], o[4] - o[1]
    trans = math.sqrt(dx * dx + dy * dy)
    rot1 = 0.0 if trans < 0.01 else wrap(math.atan2(dy, dx) - o[2])
    rot2 = wrap(wrap(o[5] - o[2]) - rot1)
    n1, n2 = rot_noise(rot1), rot_noise(rot2)
    tt, q1, q2 = trans * trans, n1 * n1, n2 * n2
    return [rot1, trans, rot2, math.sqrt(al[0] * q1 + al[1] * tt), math.sqrt((al[2] * tt + al[3] * q1) + al[3] * q2),
            math.sqrt(al[0] * q2 + al[1] * tt)]


def move(m, n3, p):
    rot1, trans, rot2, s1, st, s2 = m
    r1 = wrap(rot1 - (s1 * n3[0] if s1 > 0.0 else 0.0))
    t = trans - (st * n3[1] if st > 0.0 else 0.0)
    r2 = wrap(rot2 - (s2 * n3[2] if s2 > 0.0 else 0.0))
    a = p[2] + r1
    s, c = math.sin(a), math.cos(a)
    return [p[0] + t * c, p[1] + t * s, wrap(p[2] + wrap(r1 + r2))]


def mul33(a, b):
    out = []
    for i in range(3):
        for j in range(3):
            t = a[3 * i] * b[j]
            t = a[3 * i + 1] * b[3 + j] + t
            t = a[3 * i + 2] * b[6 + j] + t
            out.append(t)
    return out


def prior(m, p):
    s, c, t = math.sin(p[2] + m[0]), math.cos(p[2] + m[0]), m[1]
    v = [-(t * s), c, 0.0, t * c, s, 0.0, 1.0, 0.0, 1.0]
    vt = [v[0], v[3], v[6], v[1], v[4], v[7], v[2], v[5], v[8]]
    dg = [m[3] * m[3], 0.0, 0.0, 0.0, m[4] * m[4], 0.0, 0.0, 0.0, m[5] * m[5]]
    cov = mul33(mul33(v, dg), vt)
    for k in (0, 4, 8):
        cov[k] = cov[k] + EPS
    return move(m, [0.0, 0.0, 0.0], p), cov


def inv33(a):
    mi0, mi1, mi2 = a[4] * a[8] - a[7] * a[5], a[3] * a[8] - a[6] * a[5], a[3] * a[7] - a[6] * a[4]
    det = a[0] * mi0 - a[1] * mi1 + a[2] * mi2
    if det == 0.0:
        return None
    return [mi0 / det, (a[2] * a[7] - a[8] * a[1]) / det, (a[1] * a[5] - a[4] * a[2]) / det,
            -mi1 / det, (a[0] * a[8] - a[6] * a[2]) / det, (a[2] * a[3] - a[5] * a[0]) / det,
            mi2 / det, (a[1] * a[6] - a[7] * a[0]) / det, (a[0] * a[4] - a[3] * a[1]) / det]


def pose2(m, p, lm, z, n3):
    """(case, pose): 0 = still (mu), 1 = the move, 2 = the proposal (compute_proposal fs2.rs:188-216, sample_pose, set_pose)"""
    if m[3] == 0.0 and m[4] == 0.0 and m[5] == 0.0:
        return 0, move(m, [0.0, 0.0, 0.0], p)
    if not lm[2] < 100.0:
        return 1, move(m, n3, p)
    mean, cov = prior(m, p)
    dx, dy = lm[0] - mean[0], lm[1] - mean[1]
    d2 = dx * dx + dy * dy
    d = math.sqrt(d2)
    hp = [[-dx / d, -dy / d, 0.0], [dy / d2, -dx / d2, -1.0]]
    hl = [[dx / d, dy / d], [-dy / d2, dx / d2]]
    a00, a01 = hl[0][0] * lm[2] + hl[0][1] * lm[4], hl[0][0] * lm[3] + hl[0][1] * lm[5]
    a10, a11 = hl[1][0] * lm[2] + hl[1][1] * lm[4], hl[1][0] * lm[3] + hl[1][1] * lm[5]
    q00, q01 = (a00 * hl[0][0] + a01 * hl[0][1]) + R00, (a00 * hl[1][0] + a01 * hl[1][1]) + 0.0
    q10, q11 = (a10 * hl[0][0] + a11 * hl[0][1]) + 0.0, (a10 * hl[1][0] + a11 * hl[1][1]) + R11
    qdet = q00 * q11 - q10 * q01
    qi = [[1.0, 0.0], [0.0, 1.0]] if qdet == 0.0 else [[q11 / qdet, -q01 / qdet], [-q10 / qdet, q00 / qdet]]
    ppi = inv33(cov) or [(1.0 if k % 4 == 0 else 0.0) * 1e-6 for k in range(9)]
    hq = [[hp[0][i] * qi[0][j] + hp[1][i] * qi[1][j] for j in range(2)] for i in range(3)]
    pinv = [ppi[3 * i + j] + (hq[i][0] * hp[0][j] + hq[i][1] * hp[1][j]) for i in range(3) for j in range(3)]
    post = inv33(pinv) or cov
    zp1 = wrap(math.atan2(dy, dx) - mean[2])
    in0, in1 = z[0] - d, wrap(z[1] - zp1)
    for i in range(3):
        ph0, ph1 = post[3 * i] * hp[0][0], post[3 * i] * hp[1][0]
        ph0, ph1 = post[3 * i + 1] * hp[0][1] + ph0, post[3 * i + 1] * hp[1][1] + ph1
        ph0, ph1 = post[3 * i + 2] * hp[0][2] + ph0, post[3 * i + 2] * hp[1][2] + ph1
        k0, k1 = ph0 * qi[0][0] + ph1 * qi[1][0], ph0 * qi[0][1] + ph1 * qi[1][1]
        mean[i] = mean[i] + (k0 * in0 + k1 * in1)
    w = list(post)                                             # Cholesky (lower), or the square roots of the diagonal
    ok = True
    for j in range(3):
        for k in range(j):
            f = -w[3 * j + k]
            for i in range(j, 3):
                w[3 * i + j] = f * w[3 * i + k] + w[3 * i + j]
        dg = w[3 * j + j]
        if dg == 0.0 or not dg >= 0.0:
            ok = False
            break
        den = math.sqrt(dg)
        w[3 * j + j] = den
        for i in range(j + 1, 3):
            w[3 * i + j] = w[3 * i + j] / den
    low = [0.0] * 9
    if ok:
        for k in (0, 3, 4, 6, 7, 8):
            low[k] = w[k]
    else:
        for i in range(3):
            c = post[4 * i]
            low[4 * i] = math.sqrt(c if c > 0.0 else 0.0)
    out = []
    for i in range(3):
        t = low[3 * i] * n3[0]
        t = low[3 * i + 1] * n3[1] + t
        t = low[3 * i + 2] * n3[2] + t
        out.append(mean[i] + t)
    return 2, [out[0], out[1], wrap(out[2])]


ALPHAS = [[0.2, 0.2, 0.2, 0.2], [0.05, 0.01, 0.3, 0.02], [0.0, 0.0, 0.0, 0.0]]
ODOMS = [[0.0, 0.0, 0.0, 1.0, 0.2, 0.1],                                  # drive
         [3.0, -2.0, 1.2, 3.0, -2.0, 1.2],                                # stop
         [3.0, -2.0, 1.2, 3.0, -2.0, 2.9],                                # turn in place
         [3.0, -2.0, 0.3, 3.0 - 0.4 * math.cos(0.3), -2.0 - 0.4 * math.sin(0.3), 0.35],   # reverse
         [10.0, 5.0, -3.1, 10.5, 5.05, 3.1]]                              # across the wrap
POSES = [[1.0, 2.0, 0.3], [-4.0, 7.5, 3.0], [0.5, -0.25, -2.9]]
LMS = [[6.0, 4.0, 1.5, 0.1, 0.1, 2.0], [-2.0, 9.0, 0.3, 0.0, 0.0, 0.3], [0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0]]
NORMALS = [[0.3, -1.1, 0.7], [-2.0, 0.5, 1.9]]


def cases():
    out = []
    for al in ALPHAS:
        for o in ODOMS:
            m = increment(o, al)
            for p in POSES:
                mean, cov = prior(m, p)
                for n3 in NORMALS:
                    for lm in LMS:
                        dx, dy = lm[0] - p[0], lm[1] - p[1]
                        z = [math.sqrt(dx * dx + dy * dy) + 0.1 * n3[0], wrap(math.atan2(dy, dx) - p[2]) + 0.02 * n3[1]]
                        kase, q = pose2(m, p, lm, z, n3)
                        out.append({"alpha": al, "odom": o, "pose": p, "n3": n3, "lm": lm, "z": z, "increment": m,
                                    "move": move(m, n3, p), "mu": mean, "cov": cov, "case": kase, "pose2": q})
    return out


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fs_odom_golden.json")
    with open(path, "w") as f:
        json.dump({"r00": R00, "r11": R11, "eps": EPS, "cases": cases()}, f, separators=(",", ":"))
    print(path)
