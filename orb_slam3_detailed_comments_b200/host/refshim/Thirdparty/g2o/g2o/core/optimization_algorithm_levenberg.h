// refshim: Optimizer.h includes the g2o headers; the GPU-path translation unit uses none of g2o (the LM loop runs on the device), and
// Optimizer.h itself only names g2o::Sim3 in one signature.
#pragma once
namespace g2o { class Sim3; }
