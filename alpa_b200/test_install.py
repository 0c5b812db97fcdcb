"""`python -m alpa_b200.test_install` -- quick self-check of an installation (reference: alpa/test_install.py:
runs a 2-layer MLP under ShardParallel and PipeshardParallel and compares against the un-parallelised step)."""
import sys
import unittest

import torch


class InstallationTest(unittest.TestCase):
    def setUp(self):
        import alpa_b200 as alpa
        self.alpa = alpa
        import os
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:        # under torchrun: check the real (multi-node) cluster
            alpa.init(cluster="distributed")
        else:
            alpa.init(cluster="local", num_devices=4)

    def tearDown(self):
        self.alpa.shutdown()

    def _run(self, method, markers=False):
        alpa = self.alpa
        from alpa_b200.testing import assert_allclose, clone_state, get_mlp_train_state_and_step
        state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=64, num_layers=4,
                                                                add_manual_pipeline_marker=markers)
        expected, eloss = train_step(clone_state(state), batch)
        p_step = alpa.parallelize(train_step, method=method, donate_argnums=())
        actual, loss = p_step(state, batch)
        assert_allclose(expected.params, actual.params, 1e-3, 1e-3)
        assert_allclose(eloss, loss, 1e-4, 1e-4)

    def test_1_native_modules(self):
        from alpa_b200.parallel.shard.auto_sharding import planner_module
        self.assertTrue(hasattr(planner_module(), "Graph"))
        from alpa_b200 import ops
        if torch.cuda.is_available():
            self.assertTrue(ops.native_available(), "sm_90a kernels not built: python -m alpa_b200.ops.build")

    def test_2_shard_parallel(self):
        self._run(self.alpa.ShardParallel())

    def test_3_pipeline_parallel(self):
        alpa = self.alpa
        self._run(alpa.PipeshardParallel(num_micro_batches=2, layer_option=alpa.ManualLayerOption(),
                                         stage_option=alpa.UniformStageOption(num_stages=2)), markers=True)


def suite():
    s = unittest.TestSuite()
    for name in ("test_1_native_modules", "test_2_shard_parallel", "test_3_pipeline_parallel"):
        s.addTest(InstallationTest(name))
    return s


if __name__ == "__main__":
    result = unittest.TextTestRunner(verbosity=2).run(suite())
    sys.exit(0 if result.wasSuccessful() else 1)
