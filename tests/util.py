import torch


def report(name, got, ref, rtol, atol):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    nbad = int(bad.sum())
    msg = (f"{name}: max_abs_err={err.max().item():.3e} mean_abs_err={err.mean().item():.3e} "
           f"ref_abs_mean={ref.abs().mean().item():.3e} bad={nbad}/{err.numel()} (rtol={rtol}, atol={atol})")
    print(msg)
    if nbad:
        idx = bad.nonzero()[:8].tolist()
        print("  first bad idx:", idx)
        for i in idx[:4]:
            print("   ", i, float(got[tuple(i)]), float(ref[tuple(i)]))
        if got.dim() == 2:
            r, c = got.shape
            rb = bad.any(dim=1).nonzero().flatten()
            cb = bad.any(dim=0).nonzero().flatten()
            print(f"  bad rows: {rb.numel()}/{r} first {rb[:16].tolist()}; bad cols: {cb.numel()}/{c} first {cb[:16].tolist()}")
    return nbad == 0, msg


def check(name, got, ref, rtol, atol):
    ok, msg = report(name, got, ref, rtol, atol)
    assert ok, msg


# ---------------------------------------------------------------------------------------------- parity table
# Rows recorded here are printed by conftest.pytest_terminal_summary, so the measured errors of the forward-level parity
# tests appear in the test log even under `-q` (pytest captures the tests' own stdout).
PARITY_ROWS = []


def err_stats(got, ref):
    e = (got.float() - ref.float()).abs()
    return e.max().item(), e.mean().item()


def north_star_violations(got, ref, rtol=1e-3, atol=1e-4):
    """Fraction of elements outside the north star's allclose(rtol=1e-3, atol=1e-4) box."""
    e = (got.float() - ref.float()).abs()
    return (e > atol + rtol * ref.float().abs()).float().mean().item()


def record_parity(case, stage, got, ref, stock=None):
    """One row: errors of the sm_90a path and of the stock 16-bit torch execution against the same fp32 reference."""
    scale = ref.float().abs().mean().item()
    mx, mean = err_stats(got, ref)
    row = {"case": case, "stage": stage, "ref_abs_mean": scale, "ours_max": mx, "ours_mean": mean,
           "ours_viol": north_star_violations(got, ref)}
    if stock is not None:
        smx, smean = err_stats(stock, ref)
        row.update(stock_max=smx, stock_mean=smean, stock_viol=north_star_violations(stock, ref))
    PARITY_ROWS.append(row)
    return row


def assert_vs_stock(row, mean_factor=1.5, max_factor=2.0, mean_floor=2e-4, max_floor=2e-3):
    """The forward-level bar: not worse than the stock 16-bit torch stack by more than the stated factors."""
    sc = row["ref_abs_mean"]
    assert row["ours_mean"] <= mean_factor * row["stock_mean"] + mean_floor * sc, row
    assert row["ours_max"] <= max_factor * row["stock_max"] + max_floor * sc, row
