# oracle/refcli.mk — TEST INFRASTRUCTURE: the reference's own command line (src/main.cpp) on its CPU path, built as
# SURVEY §8(c) describes, into oracle/_ref/racon_cpu.  Its output is the answer of tests/golden/cli_cases.json
# (tests/golden/make_cli_cases.py) for the racon_b200 command line.  Read after oracle/Makefile, whose source lists,
# include paths and output directory it uses:
#
#   make -C oracle -f Makefile -f refcli.mk refcli
#
# Only where the reference sources exist; elsewhere a prebuilt oracle/_ref/racon_cpu is kept as it is.

.PHONY: refcli
refcli:
	@if [ -d $(REF)/src ]; then $(MAKE) -f $(HERE)Makefile -f $(HERE)refcli.mk $(REFOUT)/racon_cpu; \
	 else echo "[oracle] $(REF) absent: keeping prebuilt oracle/_ref/racon_cpu (if any)"; fi

$(REFOUT)/racon_cpu: $(REF)/src/main.cpp $(REFPOL_SRCS)
	mkdir -p $(REFOUT)
	$(CXX) -std=c++11 -O3 -mavx2 -DNDEBUG -w -DVERSION=\"1.5.0\" -Dthread_map=thread_ids $(REFPOL_INCS) -o $@ \
	  $(REF)/src/main.cpp $(REFPOL_SRCS) -lz -lpthread
