"""not-gpu: the selection and chain rules of reflectionflow_b200/tts/search.py against the reference's OWN statements.

The reference has no function for these rules: they are inline blocks of `sample()` in tts/tts_reflectionflow.py
(score -> sort -> top-k :142-182; chain init / update, best per chain, global best :358-448).  This test cuts those
statement ranges out of the reference source with `ast`, executes them in a namespace of fakes (a verifier that returns
prepared scores, an `Image` whose `open(...).save(...)` only records paths) and compares every derived quantity with
the functions used by the sharded loop, over several rounds of random scores WITH ties and duplicates (the cases where
`outputs.index`, `np.argmax` and the stable sorts decide).  What the reference statements derived is stored under
tests/golden/reference/ (tests/_refgold.py: regenerate with RF_RECORD_REFERENCE=1 and the reference tree)."""
import ast
import copy
import os
import random
import sys
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from reflectionflow_b200.tts import search as S  # noqa: E402
from tests._refgold import Store, norm, ref_path  # noqa: E402

REF = ref_path("tts/tts_reflectionflow.py")
GOLD = Store("selection_rules")


def _block(lo, hi, first_line_startswith):
    """the statements of sample() that start in source lines [lo, hi], compiled as a module"""
    src = open(REF).read()
    assert src.splitlines()[lo - 1].strip().startswith(first_line_startswith), "reference file changed"
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "sample")
    stmts = [s for s in fn.body if lo <= s.lineno <= hi]
    assert stmts
    return compile(ast.Module(stmts, []), REF, "exec")


class _Saved:
    def __init__(self, src, log):
        self.src, self.log = src, log

    def save(self, path):
        self.log.append((path, self.src))


class _FakeImage:
    def __init__(self):
        self.log = []

    def open(self, path):
        return _Saved(path, self.log)


class _FakeVerifier:
    """returns prepared per-image results in the two shapes the reference consumes"""

    def __init__(self, table):
        self.table = table  # name -> nvila ("yes"/"no", score) or openai dict

    def generate_content(self, parts):  # nvila_verifier.py:4-10 as used at :160-164
        label, score = self.table[parts[0].src]
        logits = torch.zeros(1, 2)
        logits[0, 0 if label == "yes" else 1] = score
        return label, (logits,)

    def prepare_inputs(self, images, prompts):
        return [im.src for im in images]

    def score(self, inputs, tag=None, max_new_tokens=None):
        return [copy.deepcopy(self.table[name]) for name in inputs]


def _random_results(rng, names, kind):
    vals = [round(rng.random(), 1) for _ in names]          # one decimal: many ties
    if kind == "nvila":
        return {n: ("yes" if rng.random() < 0.6 else "no", float(np.float32(0.5 + v / 2))) for n, v in zip(names, vals)}
    return {n: {"overall_score": {"score": int(10 * v), "explanation": "e"}, "accuracy_to_prompt":
                {"score": rng.randrange(11), "explanation": "x"}} for n, v in zip(names, vals)}


@pytest.mark.parametrize("kind", ["nvila", "openai"])
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_rounds_of_selection_and_chains_follow_the_reference_statements(kind, seed, tmp_path):
    rng = random.Random(seed)
    branch, rounds = 5, 4
    topk = branch if seed % 2 == 0 else branch + 2        # topk > candidates: the padding rule (:179-182)
    parents = [f"r0/{i}.png" for i in range(branch)]
    ref_chains, our_chains = {}, {}
    for rnd in range(1, rounds + 1):
        # ---- score the parents, sort, top-k: reference statements vs search.sort_outputs / select_topk
        table = _random_results(rng, parents, kind)
        names = [f"mid/{rnd}_round@{rng.randrange(10 ** 6)}.png" for _ in range(branch)]
        new_table = _random_results(rng, names, kind)
        if kind == "nvila":
            new_outputs = [{"image_name": n, "label": new_table[n][0], "score": new_table[n][1]} for n in names]
        else:
            new_outputs = [copy.deepcopy(new_table[n]) for n in names]

        def reference_round():
            ns = dict(verifier_name=kind, imagetoupdate=list(parents), verifier=_FakeVerifier(table), Image=_FakeImage(),
                      original_prompt="p", tag=None, max_new_tokens=None, choice_of_metric="overall_score",
                      yes_id=0, no_id=1, topk=topk, time=time)
            exec(_block(142, 182, "start_time = time.time()"), ns)
            # ---- new candidates, their scores, chains / best-of
            img2 = _FakeImage()
            fake_new = [_Saved(n, img2.log) for n in names]
            ns2 = dict(search_round=rnd, total_rounds=rounds, verifier_name=kind, full_imgnames=list(names),
                       chains=ref_chains, outputs=copy.deepcopy(new_outputs), choice_of_metric="overall_score",
                       selected_imgs=list(ns["selected_imgs"]), images_for_prompt=fake_new, Image=img2, np=np, os=os,
                       sample_path_lastround="last", sample_path_bestround="bestround", sample_path_best="best")
            exec(_block(358, 449, "# init chain"), ns2)
            saved = {}
            for path, src in img2.log:
                saved.setdefault(os.path.dirname(path), []).append(src)
            return {"outputs": ns["outputs"], "sorted_list": ns["sorted_list"], "selected_imgs": ns["selected_imgs"],
                    "selected_outputs": ns["selected_outputs"], "topk_idx": ns["topk_idx"],
                    "chains": ref_chains, "saved": saved}

        ref = GOLD.value(f"{kind}/seed{seed}/round{rnd}", reference_round)
        outputs = ref["outputs"]
        # the scores the reference loop collected are the ones the fake verifier returned for the parents
        if kind == "nvila":
            assert [o["score"] for o in outputs] == [table[n][1] for n in parents]
        else:
            assert outputs == norm([table[n] for n in parents])
        ours_sorted = S.sort_outputs(outputs, kind, "overall_score")
        assert norm(ours_sorted) == ref["sorted_list"]
        topk_idx, selected, selected_outputs = S.select_topk(outputs, ours_sorted, list(parents), topk)
        assert selected == ref["selected_imgs"] and norm(selected_outputs) == ref["selected_outputs"]
        assert topk_idx[:len(ref["topk_idx"])] == ref["topk_idx"]
        S.update_chains(our_chains, rnd, names, new_outputs, selected, kind, "overall_score")
        assert norm(our_chains) == ref["chains"], f"round {rnd}: chains differ"
        saved = ref["saved"]
        if rnd == 1:
            assert saved["bestround"] == names
        else:
            assert saved["bestround"] == S.best_per_chain(our_chains, kind)
        if rnd == rounds:
            assert saved["last"] == names
            assert saved["best"] == [S.global_best(our_chains, kind)]
        parents = names
