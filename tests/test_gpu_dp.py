"""Row G on real GPUs: the repo's HomographyEngine data-parallel over NCCL (needs >= 2 GPUs; run with
`python -m pytest tests/test_gpu_dp.py -m gpu` on a machine with two GPUs; it skips on one).  Asserts, for the certified tensor-core mode and the
bf16 throughput mode:
  * the gradient left by the overlapped two-phase allreduce (fc slice on the communication stream under the conv
    backward, conv slice afterwards), divided by N, equals the mean over ranks of the single-GPU gradients to 1e-5
    relative — for the fc slice and for the conv slice separately;
  * after three train steps the parameters are bit-identical on every rank;
  * one DP step equals single-GPU TF-Adam on the averaged gradient;
  * data-parallel ranks draw different dropout masks;
  * the opt-in fused multicast path (switch-side gradient sum -> sharded Adam -> multicast of the new weights and their limbs, one
    kernel) lands where the NCCL path lands, keeps the replicas' limb mirrors equal to the fp32 master, and its sharded
    Adam state gathers to identical, complete buffers.
Reference: code/utils/utils.py:380-403 (get_average_grads), code/homography_CNN_synthetic.py:199-207,277-284."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("numeric", ["bf16x3", "bf16"])
def test_engine_data_parallel_two_ranks(numeric, tmp_path):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    out = str(tmp_path / "dp.json")
    port = 29700 + (os.getpid() % 200) + (0 if numeric == "bf16" else 1)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "_dp_worker.py"), numeric, out],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.load(open(out))
    print(numeric, res)
    assert res["dropout_seeds_distinct"] and res["ranks_differ_locally"]
    # bf16x3: the two evaluations of a rank's local gradient agree to fp32-atomics noise.  Single-pass bf16 is the uncertified
    # throughput mode: its fc1 forward (split-K atomics) may flip a ReLU between two runs on identical data, 1e-3 there.
    tol = 1e-5 if numeric == "bf16x3" else 1e-3
    assert res["rel_err_fc_slice"] <= tol and res["rel_err_conv_slice"] <= tol, res
    assert res["params_bit_identical_across_ranks"] and res["params_moved"] > 0 and res["global_step"] == 3
    assert res["dp_step_vs_manual_max_update_diff_over_lr"] <= 0.02, res
    # Row G over NVSwitch multicast memory (csrc/dp_update.cu, UDH_DP_MODE=multicast): Adam's state is sharded and gathered
    # on demand, replicas stay bit-identical, and three steps land where the NCCL path lands (the switch sums in another order)
    assert res["default_path_is_nccl"] and res["nccl_engine_is_nccl"], res
    if not res["multicast_path"]:                               # opt-in mode, needs NVSwitch multicast memory
        print("multicast path not available on this box:", res.get("multicast_unavailable"))
        return
    assert res["multicast_params_bit_identical_across_ranks"], res
    assert res["adam_m_identical_after_sync"] and min(res["adam_m_fc1_nonzero_fraction_per_shard"]) > 0.02, res
    assert res["multicast_vs_nccl_rel_l2_of_update"] <= (1e-2 if numeric == "bf16x3" else 0.2), res    # three Adam steps: sign noise of near-zero gradients
    assert res.get("mirror_matches_master", True), res
