# Convenience targets (reference: Makefile targets all / test / runtest / lint; nothing here needs a configure step).
PY ?= python

.PHONY: build test test-gpu bench lint sanitize-host clean

build:            ## sm_90a CUDA extension + C++ host runtime + experimental kernels, in-tree (no GPU needed)
	$(PY) -c "import __graft_entry__ as g; g.build()"

test:             ## CPU suite (multi-process gloo tests, emulated sm100 engine, parsers, tools)
	$(PY) -m pytest tests -x -q -m "not gpu"

test-gpu:         ## on an H100
	$(PY) -m pytest tests -x -q -m gpu

bench:            ## AlexNet b=256, one GPU -> one JSON line
	$(PY) bench.py --gpus 1 --steps 20 --warmup 5

lint:
	$(PY) scripts/lint.py

sanitize-host:    ## ASan + UBSan build of csrc_host under the loader / parser / fuzz tests
	bash scripts/sanitize_host.sh asan

clean:
	rm -rf poseidon_b200/_ext/build poseidon_b200/_ext_exp/build build
