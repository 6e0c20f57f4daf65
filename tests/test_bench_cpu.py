"""CPU checks of bench.py's bookkeeping: the HBM step-roofline formula reproduces BASELINE.md §3, and the reference arm
(`--impl reference`, the oracle port on host cores) runs end to end on a tiny workload and prints the required keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bytes_per_step_matches_baseline_md():
    sys.path.insert(0, ROOT)
    import bench
    peak = 3350e9
    rows = {("llama-3.1-8b", 1): 9.69, ("llama-3.1-70b", 1): 46.72, ("llama-3.1-70b", 2): 25.96, ("llama-3.1-70b", 4): 15.58,
            ("llama-3.1-70b", 8): 10.38}
    for (t, tp), ms in rows.items():
        got = bench.bytes_per_step(t, "llama-3.2-1b", 6, 384, tp) / peak * 1e3
        assert abs(got - ms) < 0.02, (t, tp, got, ms)
    for tp, ms in ((1, 21.71), (4, 7.37)):
        q = bench.bytes_per_step("qwen3-32b", "qwen3-0.6b", 6, 384, tp) / peak * 1e3
        assert abs(q - ms) < 0.02, (tp, q, ms)


def test_reference_arm_prints_contract_keys():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "tiny",
                          "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    assert d["impl"] == "reference" and d["unit"] == "tokens/s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0


def test_usable_cores_respects_affinity_and_cgroup_quota():
    sys.path.insert(0, ROOT)
    import bench
    n = bench.usable_cores()
    assert 1 <= n <= len(os.sched_getaffinity(0))
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            assert n <= max(1, int(int(quota) / int(period)))
    except FileNotFoundError:
        pass


def test_synthetic_pair_construction():
    """The synthetic target / draft pair of the bench: both next-token maps are permutations (every greedy decision has a
    full margin), they agree on ~alpha of the tokens, the hash generator is a pure function of (stream, row, column), and
    the closed-form accept length matches a simulation of the chain the bench's parity_check walks."""
    import torch
    sys.path.insert(0, ROOT)
    from ssd_b200 import synth
    V, alpha, K = 20000, 0.85, 6
    pi_t, pi_d = synth.permutations(V, 0, alpha, "cpu")
    assert sorted(pi_t.tolist()) == list(range(V)) and sorted(pi_d.tolist()) == list(range(V))
    agree = (pi_t == pi_d).float().mean().item()
    assert abs(agree - alpha) < 0.02
    a = synth.hash_uniform(64, 256, 0.02, 5, "cpu")
    b = synth.hash_uniform(16, 256, 0.02, 5, "cpu", row0=48)
    assert torch.equal(a[48:], b) and abs(a.float().std().item() - 0.02) < 2e-3 and abs(a.float().mean().item()) < 1e-3
    assert not torch.equal(a, synth.hash_uniform(64, 256, 0.02, 6, "cpu"))
    # simulate sync SD on the chain: tokens per step = 1 + accepted prefix (truncated at K)
    tok, total, steps = 17, 0, 4000
    for _ in range(steps):
        n, cur = 0, tok
        while n < K and int(pi_d[cur]) == int(pi_t[cur]):
            cur = int(pi_t[cur])
            n += 1
        total += n + 1
        tok = int(pi_t[cur])  # the recovery token = the target's choice after the last accepted one
    assert abs(total / steps - synth.expected_tokens_per_step(alpha, K)) < 0.15
