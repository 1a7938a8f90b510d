"""TEST INFRASTRUCTURE ONLY -- CPU restatement ("oracle") of the reference hot path.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package
(``deepvoice3_pytorch_b200``) never imports it and has no CPU fallback.

Contents
--------
specs.py       layer recipes of the three reference builders, restated as flat lists
dv3_oracle.py  functional torch-CPU (fp32 or fp64) forward of every module on the path,
               driven by a reference-keyed ``state_dict`` (parity PINNED: validated against
               the live reference modules in the build container, golden vectors in
               ``tests/golden/`` made by ``tests/golden/make_golden.py``)
dropout_mask.py numpy restatement of the package's counter-based dropout mask (the package's own
               contract; pinned bit for bit to the device by tests/test_gpu_dropout.py)
audio_oracle.py numpy restatement of audio.py's STFT->linear/mel front-end
               (parity UNPINNED: lws/librosa/nnmnkwii are not vendored, see file header)
"""
