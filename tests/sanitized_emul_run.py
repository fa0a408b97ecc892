#!/usr/bin/env python
"""Runs the product's rule / encoder / single-player / replay logic (the csrc/*.cuh sources, single-lane emulation build) under
AddressSanitizer + UBSan. Usage (not part of the pytest suite; takes ~1 minute):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \
        python tests/sanitized_emul_run.py
"""
import sys, numpy as np
import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, ROOT)
import emul_lib as E
E.lib(sanitize=True)
from mortal_b200 import mjai_log, dataset_codec as DC
# 1. self-play with logging, both policies
for pol in (1, 0):
    n=24
    nonces=np.arange(123000,123000+n,dtype=np.uint64); keys=np.full(n,3,dtype=np.uint64)
    env=E.EmulEnv(nonces,keys,enable_quick_eval=(pol==1)); env.enable_log()
    acts=None
    for cyc in range(4000):
        env.step(acts)
        if cyc % 7 == 0 and env.num_rows():
            env.encode_obs(sp=True, version=4)
            if cyc % 21 == 0: env.encode_obs(sp=False, version=2)
        acts=env.policy_test(pol)
        if env.num_live()==0: break
    words,lens=env.read_log(); env.close()
    games=[[{"type":"start_game","names":["a","b","c","d"],"seed":[int(nonces[t]),3]}]+mjai_log.decode_events(words[t,:int(lens[t])])+[{"type":"end_game"}] for t in range(n)]
    # 2. replay with encode
    jobs=DC.build_jobs(games[:8],[[0,1,2,3]]*8)
    rep=E.EmulReplay(jobs)
    for it in range(3000):
        rep.replay_step()
        if rep.num_rows() and it % 5 == 0: rep.encode_obs(sp=True, version=4)
        if rep.live==0: break
    assert (rep.errs()==0).all()
    rep.close()
    print("policy",pol,"ok cycles",cyc,"replay iters",it, flush=True)
# 3. batch runner with guard
r=E.run(np.arange(5000,5200,dtype=np.uint64),np.full(200,9,dtype=np.uint64),policy_kind=1,quick_eval=True,agari_guard=True,trace_cap=1<<20)
assert (r["errs"]==0).all()
print("sanitised run finished")
