# tests/native/ref_partition.mk — test infrastructure: builds tests/native/ref_compact_partition.cc (the reference driver with the
# partitioner options) with oracle/Makefile's flags, next to the driver it wraps:
#   make -C oracle -f ../tests/native/ref_partition.mk partition
include Makefile
SELF := ../tests/native/ref_partition.mk
PART_SRC := ../tests/native/ref_compact_partition.cc

.PHONY: partition
partition:
	@if [ -d $(REF)/db ]; then $(MAKE) -f $(SELF) $(OUT)/ref_compact_partition && \
	  if [ -f $(B200_LIB_DIR)/libb200c.so ]; then $(MAKE) -f $(SELF) $(OUT)/ref_compact_partition_b200; fi; \
	else echo "no $(REF): using prebuilt $(OUT)/ if present"; fi

$(OUT)/ref_compact_partition: $(PART_SRC) ref_compact.cc $(OUT)/libtoplingdb_ref.so
	$(CXX) $(REF_CXXFLAGS) -I$(CURDIR)/.. -o $@ $(PART_SRC) -L$(OUT) -ltoplingdb_ref -Wl,-rpath,'$$ORIGIN' -pthread -ldl

$(OUT)/ref_compact_partition_b200: $(PART_SRC) ref_compact.cc $(PLUGIN_SRCS) $(PLUGIN_HDRS) $(OUT)/libtoplingdb_ref.so $(B200_LIB_DIR)/libb200c.so
	$(CXX) $(REF_CXXFLAGS) -DWITH_B200_PLUGIN -I$(CURDIR)/.. -I$(CURDIR)/../include -o $@ $(PART_SRC) \
	  $(PLUGIN_SRCS) -L$(OUT) -ltoplingdb_ref -L$(B200_LIB_DIR) -lb200c \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../toplingdb_b200' -pthread -ldl
