"""The measurement contract that can be checked without a GPU: `bench.py --impl reference` prints exactly ONE JSON line on stdout with the
keys the driver reads (everything else -- constructor prints of the reference, library banners -- goes to stderr), and the ncu
family classifier of tools/ncu_traffic.py maps the shipped kernels' names to the families bench.py reports."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout[:500]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "images/sec" and d["higher_is_better"] is True and d["value"] > 0
    assert d["metric"] == "PartialConv UNet 512x512 images/sec (fwd+bwd)" and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "images/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and d["gpu_launches"] == 0


def test_ncu_family_classifier_knows_the_shipped_kernels():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from ncu_traffic import family
    finally:
        sys.path.pop(0)
    u = "void <unnamed>::"
    assert family(u + "pconv_tc_tma_kernel<64, 0, 1, 0>(<unnamed>::TcParams, CUtensorMap_st)") == "tc_fwd"
    assert family(u + "pconv_tc_tma_kernel<(int)256, (int)1, (bool)0, (bool)0>(TcParams)") == "tc_dgrad"
    assert family(u + "pconv_tc_sp_kernel<(int)64>(<unnamed>::TcParams, <unnamed>::SpTable, CUtensorMap_st, CUtensorMap_st)") == "tc_dgrad"
    assert family(u + "pconv_tc_wgrad_tma_kernel<64, 4, 1>(WgParams)") == "tc_wgrad"
    assert family(u + "k2r_combine_kernel<3>(K2rParams)") == "tc_fwd"
    assert family(u + "k2r_dbuild_kernel<0, 3>(K2rParams)") == "tc_dgrad"
    assert family(u + "k2r_dbuild_kernel<1, 3>(K2rParams)") == "tc_wgrad"
    assert family(u + "dw4_s1_kernel<__nv_bfloat16, 0>(const T1 *)") == "dw_fwd"
    assert family(u + "dw4_s1_kernel<__nv_bfloat16, (bool)1>(const T1 *)") == "dw_dgrad"
    assert family(u + "dw4_s1_wgrad_kernel<__nv_bfloat16>(const T1 *)") == "dw_wgrad"
    assert family(u + "bn_fwd_fused_kernel<__nv_bfloat16, 2>(...)") is None
