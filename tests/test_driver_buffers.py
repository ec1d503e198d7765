"""The device buffers of the host drivers (bwag_api.cu and the per-command drivers) are all returned: after mem_process_seqs
has run many batches, with every optional kernel that has scratch of its own switched on, closing the index (which destroys
its device context) leaves as many live device blocks as there were before it was opened.  The emulator build of the drivers
counts the blocks of cudaMalloc and cudaFree (bwag_drv.h); a batch object that is freed, whether at bwag_batch_end or with its
context, must take all of its own with it."""
import ctypes as C
import os
import re

from conftest import ROOT

CUSIM_SO = os.path.join(ROOT, "tests", "_build", "libbwa_b200_cusim.so")


def test_context_and_batches_free_every_device_block(data, monkeypatch, capfd):
    import bwa_b200
    L = bwa_b200.lib(CUSIM_SO)
    L.bwag_cusim_live_dev_blocks.restype = C.c_long
    fa, (fq,) = data.reads("c1", tag="drvbuf", n=1120, seed=41)
    monkeypatch.setenv("BWA_B200_SELFCHECK", "0")
    monkeypatch.setenv("BWA_B200_PROFILE", "1")
    monkeypatch.setenv("BWA_B200_K5_LANE", "1")   # K5L (lane-per-request global alignment) and its scratch
    monkeypatch.setenv("BWA_B200_CHUNK", "80")    # 14 batches, more than the context keeps for reuse (12)
    monkeypatch.setenv("BWA_B200_LANES", "2")
    before = L.bwag_cusim_live_dev_blocks()
    idx = bwa_b200.Index(fa, library=L)
    batch = bwa_b200.ReadBatch(fq, library=L)
    bwa_b200.mem_process_seqs(L.mem_opt_init(), idx, batch)
    assert batch.sam().count(b"\n") >= 1120
    assert L.bwag_cusim_live_dev_blocks() > before
    idx.close()
    err = capfd.readouterr().err
    assert len(re.findall(r"lane-per-request kernel made [1-9]\d* of (\d+)", err)) >= 14, err[-2000:]
    assert L.bwag_cusim_live_dev_blocks() == before
