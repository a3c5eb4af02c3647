# Convenience targets; the Python entry points (__graft_entry__.build, solo_b200.build) do the same work.
PY ?= python

.PHONY: lib oracle hostsim test-cpu test-gpu bench clean
lib:            ## solo_b200/libsolo_b200.so (nvcc, sm_90a)
	$(PY) -m solo_b200.build
oracle:         ## the unmodified reference compiled into oracle/_ref (needs /root/reference)
	$(MAKE) -C oracle -j4
hostsim:        ## host build of the kernel source used by the CPU test-suite
	$(PY) -c "from tests.hostsim import build_hostsim as b; b.build(); b.build(emu=True)"
test-cpu: lib hostsim
	$(PY) -m pytest tests -q -m "not gpu"
test-gpu: lib
	$(PY) -m pytest tests -q -m gpu
bench: lib
	$(PY) bench.py
clean:
	rm -rf solo_b200/libsolo_b200.so tests/_hostsim oracle/_ref variants
