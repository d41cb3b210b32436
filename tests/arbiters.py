"""Independent arbiters for the CPU oracle (TEST INFRASTRUCTURE): textbook formulas evaluated with mpmath at 40 or 50 digits, scipy's
root finder / interpolator — nothing here shares code, recursions or operation order with oracle/ or nyx_b200/.

Spherical-harmonic acceleration (Vallado, *Fundamentals of Astrodynamics*, eq. 8-19/8-27; Montenbruck & Gill eq. 3.27-3.33):
    U = (mu / r) sum_{n>=1} sum_{m<=n} (R / r)^n  Pbar_nm(sin phi) (Cbar_nm cos m lam + Sbar_nm sin m lam)
    a_r   = -(mu / r^2) sum (n + 1) (R/r)^n Pbar_nm (C cos + S sin)
    a_phi =  (mu / r^2) sum (R/r)^n dPbar_nm/dphi (C cos + S sin),   dP_nm/dphi = P_{n,m+1} - m tan(phi) P_nm
    a_lam =  (mu / (r^2 cos phi)) sum (R/r)^n m Pbar_nm (S cos - C sin)
with geodesy's normalisation Pbar = sqrt((2 - delta_0m)(2n + 1)(n - m)! / (n + m)!) P and no Condon-Shortley phase.  The fully
normalised functions Pbar_nm(sin phi) come from one of two sources:
  closed     the associated Legendre FUNCTIONS from their closed (hypergeometric) form, `mpmath.legenp`, no recursion, 40 digits
             (mp_harmonic_accel); about 150 s per point at degree 96 on one core
  recursion  the standard forward-column recursion of Holmes & Featherstone (2002), eq. 11-13, 50 digits
             (mp_harmonic_accel_recursion): the sectoral seeds Pbar_mm = sqrt((2m + 1) / 2m) cos(phi) Pbar_{m-1,m-1} (Pbar_11 =
             sqrt(3) cos phi), then Pbar_nm = a_nm sin(phi) Pbar_{n-1,m} - b_nm Pbar_{n-2,m} down each column.  Checked against
             the closed form to 1e-25 (tests/test_high_degree_inputs.py); a fraction of a second per point at degree 96."""
import mpmath as mp


def _pbar_closed(n, mtop, sphi):
    """Pbar_n0 .. Pbar_n,mtop (sin phi) from the closed form"""
    out = []
    for m in range(0, mtop + 1):
        # mpmath's type-2 function carries the Condon-Shortley phase (-1)^m: remove it
        norm = mp.sqrt((2 if m else 1) * (2 * n + 1) * mp.factorial(n - m) / mp.factorial(n + m))
        out.append(norm * ((-1) ** m) * mp.legenp(n, m, sphi))
    return out


def _pbar_recursion(degree, sphi, cphi):
    """rows P[n][m], m = 0..n, of the fully normalised functions by the forward-column recursion"""
    P = [[mp.mpf(0)] * (n + 1) for n in range(degree + 1)]
    P[0][0] = mp.mpf(1)
    for m in range(0, degree + 1):
        if m == 1:
            P[1][1] = mp.sqrt(3) * cphi
        elif m > 1:
            P[m][m] = mp.sqrt(mp.mpf(2 * m + 1) / (2 * m)) * cphi * P[m - 1][m - 1]
        for n in range(m + 1, degree + 1):
            a = mp.sqrt(mp.mpf((2 * n - 1) * (2 * n + 1)) / ((n - m) * (n + m)))
            b = mp.sqrt(mp.mpf((2 * n + 1) * (n + m - 1) * (n - m - 1)) / ((n - m) * (n + m) * (2 * n - 3))) if n >= m + 2 else 0
            P[n][m] = a * sphi * P[n - 1][m] - (b * P[n - 2][m] if n >= m + 2 else 0)
    return P


def _accel(c_nm, s_nm, degree, order, mu, r_eq, rb, dps, legendre, as_mpf):
    mp.mp.dps = dps
    x, y, z = (mp.mpf(float(v)) for v in rb)
    r = mp.sqrt(x * x + y * y + z * z)
    sphi = z / r
    cphi = mp.sqrt(x * x + y * y) / r
    tphi = sphi / cphi
    lam = mp.atan2(y, x)
    mu, r_eq = mp.mpf(float(mu)), mp.mpf(float(r_eq))
    rows = _pbar_recursion(degree, sphi, cphi) if legendre == "recursion" else None
    ar = aphi = alam = mp.mpf(0)
    for n in range(1, degree + 1):
        rn = (r_eq / r) ** n
        mtop = min(n, order)
        top = min(mtop + 1, n)
        # Pbar_n0 .. Pbar_n,mtop+1 (Pbar_n,n+1 = 0)
        P = (rows[n][: top + 1] if rows else _pbar_closed(n, top, sphi)) + [mp.mpf(0)]
        for m in range(0, mtop + 1):
            c, s = mp.mpf(float(c_nm[n][m])), mp.mpf(float(s_nm[n][m]))
            if c == 0 and s == 0:
                continue
            cs = c * mp.cos(m * lam) + s * mp.sin(m * lam)
            sc = s * mp.cos(m * lam) - c * mp.sin(m * lam)
            # dPbar_nm / dphi from the unnormalised rule: Pbar_n,m+1 carries norm(n, m+1), and
            # norm(n, m)^2 / norm(n, m+1)^2 = (2 - delta_0m) / 2 (n - m)(n + m + 1)
            ratio = mp.sqrt(mp.mpf(2 if m else 1) / 2 * (n - m) * (n + m + 1))
            dP = ratio * P[m + 1] - m * tphi * P[m]
            ar -= (n + 1) * rn * P[m] * cs
            aphi += rn * dP * cs
            alam += rn * m * P[m] * sc
    k = mu / (r * r)
    ar, aphi, alam = k * ar, k * aphi, k * alam / cphi
    # spherical -> Cartesian (unit vectors e_r, e_phi, e_lam)
    cl, sl = mp.cos(lam), mp.sin(lam)
    ax = ar * cphi * cl - aphi * sphi * cl - alam * sl
    ay = ar * cphi * sl - aphi * sphi * sl + alam * cl
    az = ar * sphi + aphi * cphi
    return (ax, ay, az) if as_mpf else (float(ax), float(ay), float(az))


def mp_harmonic_accel(c_nm, s_nm, degree, order, mu, r_eq, rb, dps=40, as_mpf=False):
    """Non-central acceleration [km/s^2] at the body-fixed position rb [km] (three floats) for normalised coefficients
    c_nm[n][m], s_nm[n][m], closed-form Legendre functions; three Python floats rounded from `dps`-digit arithmetic (as_mpf: the
    mpmath values)."""
    return _accel(c_nm, s_nm, degree, order, mu, r_eq, rb, dps, "closed", as_mpf)


def mp_harmonic_accel_recursion(c_nm, s_nm, degree, order, mu, r_eq, rb, dps=50, as_mpf=False):
    """The same acceleration with the Legendre functions from the Holmes & Featherstone forward-column recursion."""
    return _accel(c_nm, s_nm, degree, order, mu, r_eq, rb, dps, "recursion", as_mpf)


def sun_visible_fraction(r_ls, r_body, d, n=1500):
    """Fraction of a disk of angular radius r_ls (light source) NOT covered by a disk of angular radius r_body whose centre is the
    angle d away, by brute-force area quadrature on a polar grid (small-angle, planar geometry: what `occultation` models)."""
    import numpy as np

    rr = (np.arange(n) + 0.5) / n * r_ls
    th = (np.arange(2 * n) + 0.5) / (2 * n) * 2 * np.pi
    R, T = np.meshgrid(rr, th, indexing="ij")
    px, py = R * np.cos(T), R * np.sin(T)
    covered = (px - d) ** 2 + py ** 2 < r_body ** 2
    w = R   # area element r dr dtheta (constant factors cancel in the ratio)
    return 1.0 - float((w * covered).sum() / w.sum())
