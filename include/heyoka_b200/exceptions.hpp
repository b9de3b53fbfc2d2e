// heyoka_b200 — exception types of the C++ API.
#ifndef HEYOKA_B200_EXCEPTIONS_HPP
#define HEYOKA_B200_EXCEPTIONS_HPP

#include <stdexcept>

namespace heyoka_b200
{

// include/heyoka/exceptions.hpp:19.
struct not_implemented_error final : std::runtime_error {
    using std::runtime_error::runtime_error;
};

} // namespace heyoka_b200

#endif
