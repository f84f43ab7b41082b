"""Data-parallel correctness on real GPUs (needs >= 2; skipped on a one-GPU box): tools/dp_check.py under torchrun --
NCCL through the C-ABI communicator, DP step == single-GPU step on replicated data, bit-identical parameters across ranks on sharded
data, the reference's parameter averaging (J:325-330), sync_bn "W x N/W == 1 x N" (SURVEY.md 8e), bf16 gradient payload, and the
overlapped two-bucket all-reduce."""
import os

import pytest

from helpers import run_two_ranks

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("overlap,p2p", [("0", "1"), ("0", "0"), ("1", "0")], ids=["peer-memory all-reduce", "nccl", "nccl two-bucket overlap"])
def test_two_rank_data_parallel(overlap, p2p, tmp_path):
    env = dict(os.environ, B2G_AR_OVERLAP=overlap, B2G_P2P_AR=p2p)
    d = run_two_ranks("dp_check.py", tmp_path / "dp_check_rank0.json", 29531 + int(overlap) + 2 * int(p2p), env=env, timeout=900)
    assert d["world"] == 2 and d["allreduce"] == "ok" and d["ar_overlap_env"] == overlap
    assert d["allreduce_transport"] == ("peer-memory kernel" if p2p == "1" else "nccl"), d["allreduce_transport"]
    for k in ("sharded_fp32_G_identical", "sharded_fp32_D_identical", "sharded_bf16_G_identical", "sharded_bf16_D_identical", "bf16_payload_G_identical", "bf16_payload_D_identical"):
        assert d[k] is True, k
    assert d["parameter_averaging_max_abs_err"] < 1e-6
    assert d["sync_bn"]["max_abs_dG"] < 4.5e-3 and d["sync_bn"]["max_abs_dD"] < 4.5e-3 and d["sync_bn"]["mean_abs_dG"] < 5e-5 and d["sync_bn"]["mean_abs_dD"] < 5e-5
