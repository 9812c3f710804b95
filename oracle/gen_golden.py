#!/usr/bin/env python
"""Generate tests/golden/ from the UNMODIFIED reference (oracle/_ref/libref_seq.so).

TEST INFRASTRUCTURE ONLY.  Run in the authoring container (needs /root/reference to have been compiled by
`make -C oracle`).  The reference ships no tests or golden vectors (SURVEY.md section 4), so every fixture is an
output of the reference's own code on real MNIST bytes:

  mnist_subset.npz       first 1024 training and first 256 test samples, raw u8 + labels (the IDX payload bytes)
  reference_vectors.npz  seed-1 parameters, per-sample activations / backward buffers, parameter states after
                         1, 1000 and 60000 steps, per-step error norms, classifications
  reference_scalars.json the SURVEY.md Appendix B numbers re-measured here (err, error rate, sums, FNV hashes)
  reference_ops_random.json SHA-256 of the bits of every operator of layer.h on seeded random inputs (oracle_lib.ops_chain)

`gen_golden.py ops` writes only reference_ops_random.json.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import oracle_lib as O  # noqa: E402

N_TRAIN_SUB, N_TEST_SUB = 1024, 256


def ops_golden(ref):
    digests = {k: O.bits_digest(v) for k, v in O.ops_chain(ref, reference=True).items()}
    with open(os.path.join(O.GOLDEN, "reference_ops_random.json"), "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)


def main():
    ref = O.reference()
    if ref is None:
        raise SystemExit("oracle/_ref/libref_seq.so missing: run `make -C oracle` where the reference sources exist")
    ops_golden(ref)
    if sys.argv[1:] == ["ops"]:
        return
    data = O.full_mnist()
    if data is None:
        raise SystemExit("oracle/_ref/data missing")
    tr, trl, te, tel = data
    os.makedirs(O.GOLDEN, exist_ok=True)
    np.savez_compressed(os.path.join(O.GOLDEN, "mnist_subset.npz"),
                        train_u8=tr[:N_TRAIN_SUB], train_labels=trl[:N_TRAIN_SUB],
                        test_u8=te[:N_TEST_SUB], test_labels=tel[:N_TEST_SUB])

    def params():
        p = np.empty(O.NPARAM, np.float32)
        ref.ref_get_params(O.fp(p))
        return p

    def acts():
        a = np.empty(O.N_ACTS, np.float32)
        ref.ref_get_acts(O.fp(a))
        return a

    def back():
        b = np.empty(7520 + 2160, np.float32)
        ref.ref_get_back(O.fp(b))
        return b

    out = {}
    sc = {}
    ref.ref_reset_params()
    p0 = params()
    out["params_init"] = p0
    # forward records for the first 8 samples with the seed-1 parameters
    fa = []
    for s in range(8):
        ref.ref_forward_u8(O.u8p(tr[s]))
        fa.append(acts())
    out["acts_init_first8"] = np.stack(fa)
    # step-by-step: backward record of step 1, error norms of the first 1000 steps
    errs = np.empty(1000, np.float32)
    for s in range(1000):
        errs[s] = ref.ref_train_step_u8(O.u8p(tr[s]), int(trl[s]))
        if s == 0:
            out["back_step1"] = back()
            out["acts_step1"] = acts()
            out["params_after1"] = params()
    out["err_first1000"] = errs
    out["params_after1000"] = params()
    out["pred_test_sub_after1000"] = np.array([ref.ref_classify_u8(O.u8p(te[s])) for s in range(N_TEST_SUB)], np.uint8)
    out["wrong_test_sub_after1000"] = np.array(ref.ref_test_u8(O.u8p(te[:N_TEST_SUB].reshape(-1)), O.u8p(tel[:N_TEST_SUB]), N_TEST_SUB))
    # continue to 20,000 then a full epoch from scratch through the driver-shaped loop
    ref.ref_reset_params()
    secs = np.zeros(1, np.float64)
    e20k = ref.ref_learn_loop_u8(O.u8p(tr[:20000].reshape(-1)), O.u8p(trl[:20000]), 20000, O.dp(secs))
    sc["mean_err_first_20000"] = float(e20k)
    ref.ref_reset_params()
    e_epoch = ref.ref_learn_loop_u8(O.u8p(tr.reshape(-1)), O.u8p(trl), 60000, O.dp(secs))
    sc["epoch_err"] = float(e_epoch)
    sc["epoch_err_printed"] = "%e" % e_epoch
    sc["epoch_seconds_here"] = float(secs[0])
    out["params_after_epoch"] = params()
    wrong = int(ref.ref_test_u8(O.u8p(te.reshape(-1)), O.u8p(tel), 10000))
    sc["test_wrong_after_epoch"] = wrong
    sc["test_error_rate_printed"] = "%.2lf%%" % (wrong / 10000.0 * 100.0)
    out["pred_test_sub_after_epoch"] = np.array([ref.ref_classify_u8(O.u8p(te[s])) for s in range(N_TEST_SUB)], np.uint8)

    def sums(p, tag):
        for k, (a, b) in O.OFF.items():
            sc[f"{tag}.sum.{k}"] = float(np.sum(p[a:b].astype(np.float64)))
        sc[f"{tag}.fnv.c1w"] = "%08x" % O.fnv1a32(p[0:150])
        sc[f"{tag}.fnv.fw"] = "%08x" % O.fnv1a32(p[173:2333])

    sums(p0, "init")
    sums(out["params_after1"], "after1")
    sums(out["params_after1000"], "after1000")
    sums(out["params_after_epoch"], "after_epoch")
    sc["sample0.err"] = float(errs[0])
    sc["sizeof_mnist_data"] = int(ref.ref_sizeof_mnist_data())
    np.savez_compressed(os.path.join(O.GOLDEN, "reference_vectors.npz"), **out)
    with open(os.path.join(O.GOLDEN, "reference_scalars.json"), "w") as f:
        json.dump(sc, f, indent=1, sort_keys=True)
    print(json.dumps(sc, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
