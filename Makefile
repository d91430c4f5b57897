# libalq.so (CUDA, sm_90a).  `make` == `python -m active_learning_b200.build`
PY ?= python

all:
	$(PY) -m active_learning_b200.build

force:
	$(PY) -m active_learning_b200.build --force

clean:
	rm -rf active_learning_b200/csrc/_obj active_learning_b200/libalq.so

test:
	$(PY) -m pytest tests -x -q -m "not gpu"

.PHONY: all force clean test
