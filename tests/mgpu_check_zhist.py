"""RedshiftHistogram on every GPU of the box (torchrun, one process per GPU) against one GPU and the oracle: Scott's
edges bit-identical on every rank and within 1e-13 of one GPU, counts equal on the same edges, weighted sums, and the
'raise' interpolation raising on every rank together.

    torchrun --nproc-per-node 2 tests/mgpu_check_zhist.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from nbodykit_b200 import comm as C
    from nbodykit_b200.cosmology import Planck15
    from nbodykit_b200.lab import ArrayCatalog, RedshiftHistogram
    from oracle import zhist_oracle as zo
    world = C.world()
    P, rank = world.size, world.rank
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    z = zo.make_redshifts(23, 400000)
    w = np.random.RandomState(4).uniform(size=z.size)
    n = z.size
    mine = slice(rank * n // P, (rank + 1) * n // P)
    edges = np.r_[0.0, np.cumsum(np.random.RandomState(5).uniform(0.5, 1.5, 300))] / 300.
    for bins in (None, 40, edges):
        for weighted in (False, True):
            cols = {"z": torch.from_numpy(z[mine]).cuda()}
            if weighted:
                cols["w"] = torch.from_numpy(w[mine]).cuda()
            r = RedshiftHistogram(ArrayCatalog(cols, comm=world), 0.15, Planck15, bins=bins, redshift="z",
                                  weight="w" if weighted else None)
            all_edges = world.allgather(r.bin_edges)
            assert all(np.array_equal(e, r.bin_edges) for e in all_edges), "edges differ between ranks"
            got = r.nbar * r.dV
            want = zo.counts(z, r.bin_edges, w if weighted else None)
            if weighted:
                assert (np.abs(got - want) <= 1e-12 * zo.counts(z, r.bin_edges, w) + 1e-300).all(), "weighted sums"
            else:
                assert np.array_equal(np.rint(got), want) and np.array_equal(r.nbar, want / r.dV), "counts"
            if rank == 0:
                one = RedshiftHistogram(ArrayCatalog({"z": torch.from_numpy(z).cuda()}, comm=C.SelfComm()), 0.15, Planck15,
                                        bins=bins, redshift="z")
                assert len(one.bin_edges) == len(r.bin_edges)
                np.testing.assert_allclose(r.bin_edges, one.bin_edges, rtol=1e-13, atol=0)
            world.barrier()
        try:
            r.interpolate(np.array([9.0 if rank == P - 1 else 0.5]), "raise")
            raised = False
        except ValueError:
            raised = True
        assert all(world.allgather(raised)), "'raise' did not raise on every rank"
        if rank == 0:
            print("mgpu_check_zhist ok: %d GPUs, %d rows, bins %s, %d bins" % (P, n, "Scott" if bins is None else
                                                                             ("int" if np.isscalar(bins) else "explicit"),
                                                                             len(r.bin_edges) - 1))
        world.barrier()


if __name__ == "__main__":
    main()
