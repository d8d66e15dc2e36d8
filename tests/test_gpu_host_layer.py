"""GPU tier: the host-buffer batch calls keep one pipeline cache per thread, keyed by device and shape.  A shape cached by
the single-device call is reused by the _multi call on the same device (no second pipeline), and after b200z_init(1) a
single-device batch of a shape cached on device 0 gets a pipeline on device 1."""
import pytest

from sharpziplib_b200 import datagen

pytestmark = pytest.mark.gpu


def test_batch_entry_points_share_one_pipeline_cache(z):
    import torch
    bufs = [datagen.silesia_mix(i, 1 << 20).tobytes() for i in range(64)]
    plan = z.DeflatePlan([len(b) for b in bufs], level=6)
    ws = plan.workspace_bytes
    plan.close()
    z.lib().b200z_release_cached()
    try:
        outs, _ = z.deflate_batch(bufs, level=6)
        free_before = torch.cuda.mem_get_info(0)[0]
        outs_multi, _ = z.deflate_batch(bufs, level=6, devices=[0])
        free_after = torch.cuda.mem_get_info(0)[0]
        assert outs_multi == outs
        # (half a workspace of slack: other processes may share the card)
        assert free_before - free_after < ws // 2, "the _multi call built a second pipeline for a shape already cached on device 0"
        if torch.cuda.device_count() >= 2:
            z.init(1)
            free_before = torch.cuda.mem_get_info(1)[0]
            outs_dev1, _ = z.deflate_batch(bufs, level=6)
            free_after = torch.cuda.mem_get_info(1)[0]
            assert outs_dev1 == outs
            assert free_before - free_after >= ws // 2, "after init(1) the batch reused the pipeline cached on device 0"
    finally:
        z.lib().b200z_release_cached()
        z.init(0)
