# TEST INFRASTRUCTURE ONLY: _ref/libmodbase_ref.so, the reference's modified-base config and model code
# (config/ModBaseModelConfig.cpp, modbase/nn/ModBaseModel.cpp) compiled unmodified where they lie, plus the C-ABI shim
# modbase_ref_driver.cpp.  Linked against _ref/libdorado_ref.so (the Makefile in this directory), which provides the
# ConvStack / LSTMStack / LinearUpsample modules, config::common and the torch utilities those sources call.
# Only built where the reference tree exists; the built library travels with the tree.
#   make -C oracle -f modbase_ref.mk
include Makefile

MB_SRCS := config/ModBaseModelConfig.cpp modbase/nn/ModBaseModel.cpp
MB_OBJS := $(patsubst %.cpp,$(OBJ)/%.o,$(MB_SRCS))

.DEFAULT_GOAL := modbase_ref
.PHONY: modbase_ref

ifneq ($(wildcard $(D)/modbase/nn/ModBaseModel.cpp),)
modbase_ref: $(OUT)/libmodbase_ref.so $(OUT)/modbase_host

# -I$(D)/modbase: ModBaseModel.cpp includes its own header as "ModBaseModel.h"
$(OUT)/libmodbase_ref.so: $(MB_OBJS) $(OBJ)/modbase_ref_driver.o $(OUT)/libdorado_ref.so
	$(CXX) -shared -o $@ $(MB_OBJS) $(OBJ)/modbase_ref_driver.o -L$(OUT) -ldorado_ref $(LDFLAGS_REF) -Wl,-rpath,'$$ORIGIN'

# The reference-side binding (include/B200ModBaseModel.h) compiled against the reference's headers and EXECUTED: a host
# program that builds the module as load_modbase_model would and runs its forward (modbase_host.cpp; run by
# tests/test_modbase_gpu.py).  Needs ../dorado_b200/libb200call.so.
$(OUT)/modbase_host: modbase_host.cpp ../include/B200ModBaseModel.h ../include/b200call.h $(OUT)/libmodbase_ref.so
	$(CXX) $(CXXFLAGS) -I../include modbase_host.cpp -o $@ -L$(OUT) -lmodbase_ref -ldorado_ref -L../dorado_b200 -lb200call \
	  $(LDFLAGS_REF) -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../dorado_b200'

$(OBJ)/modbase_ref_driver.o: modbase_ref_driver.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -I$(D)/modbase -c $< -o $@
else
modbase_ref:
	@echo "reference tree $(REF) not present: keeping prebuilt $(OUT)/libmodbase_ref.so (if any)"
endif
