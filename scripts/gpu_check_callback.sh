python -m pytest tests -m gpu -x -q 2>&1 | tail -25
python - <<'PY'
import mrcal_b200, numpy as np
from mrcal_b200 import synthetic
for c in (2,3):
    kw,_ = synthetic.baseline_config(c)
    P = mrcal_b200.Problem(**kw)
    print('config',c,'callback ms with J', P.time_callback(20,True), 'no J', P.time_callback(20,False), 'nnz', P.N_j_nonzero)
PY
python -c 'import sys; sys.path.insert(0, "scripts"); import measure; print(measure.card())'
