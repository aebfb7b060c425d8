"""Golden DotProductProofLog proofs at the sizes whose oracle run takes minutes (the oracle folds the generators pair by pair, about 100 us per pair
on a CPU): n = 2^18 and 2^20 by default.  For each n: gens DotProductProofGens::new(n, b"dotlog-golden"), x = prg_scalars("dotlog-golden-x-<logn>", n),
a = prg_scalars("dotlog-golden-a-<logn>", n), blind_x, blind_y = prg_scalars("dotlog-golden-blinds-<logn>", 2), y = <x, a>, transcript
Transcript(b"dotlog-golden") and tape RandomTape(b"proof", tape_seed(logn)).  Writes tests/golden/dotlog_golden.json {logn: {proof, Cx, Cy, y,
transcript_after, tape_after}} (hex; *_after = 64 challenge bytes labelled b"after" drawn from the states the prove left).
    python tests/golden/make_dotlog_golden.py [logn ...]"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.spartan_ref import core as oc
from oracle.spartan_ref import protocol as pr
from oracle.spartan_ref import r1cs

LABEL, GENS_LABEL = b"dotlog-golden", b"dotlog-golden"
OUT = os.path.join(ROOT, "tests", "golden", "dotlog_golden.json")


def case(logn):
    n = 1 << logn
    x = oc.prg_scalars("dotlog-golden-x-%d" % logn, n)
    a = oc.prg_scalars("dotlog-golden-a-%d" % logn, n)
    blind_x, blind_y = oc.to_ints(oc.prg_scalars("dotlog-golden-blinds-%d" % logn, 2))
    xi, ai = oc.to_ints(x), oc.to_ints(a)
    y = sum(p * q for p, q in zip(xi, ai)) % oc.Q
    gens = pr.DotProductProofGens(n, GENS_LABEL)
    T, tape = oc.Transcript(LABEL), oc.RandomTape(b"proof", r1cs.tape_seed(logn))
    proof, Cx, Cy = pr.DotProductProofLog.prove(gens, T, tape, xi, blind_x, ai, y, blind_y)
    return {"proof": pr.ser(proof).hex(), "Cx": Cx.hex(), "Cy": Cy.hex(), "y": "%064x" % y,
            "transcript_after": T.challenge_bytes(b"after", 64).hex(), "tape_after": tape.tape.challenge_bytes(b"after", 64).hex()}


def main():
    oc.lib.oracle_set_threads(os.cpu_count() or 1)
    logns = [int(v) for v in sys.argv[1:]] or [18, 20]
    out = json.load(open(OUT)) if os.path.exists(OUT) else {}
    for logn in logns:
        t0 = time.time()
        out[str(logn)] = case(logn)
        json.dump(out, open(OUT, "w"), indent=1, sort_keys=True)
        print("2^%d: %.0f s" % (logn, time.time() - t0), flush=True)


if __name__ == "__main__":
    main()
